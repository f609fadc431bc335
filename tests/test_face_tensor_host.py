"""CPU: face tensors (DESIGN.md 2, "Face crops", item 6) through the host build of k_face_crop's per-tensor code
(ht_selftest_face_tensor) and of its per-pixel conversion (ht_selftest_tensor_pixels), against the independent C
restatement tests/crop_tensor_oracle.c, numpy and exact rationals:

  * every byte value x every dtype x a set of (mul, add) - torchvision's ImageNet constants, tiny and huge values, and
    values that overflow f16 and bf16 - converts as the restatement does, bit for bit; f32 is the exactly rounded
    c mul + add (fractions), f16 is numpy's f32 -> f16 of it and bf16 its round-to-nearest-even; against torchvision's
    two-step fp32 (x / 255 - mean) / std it is within the bound stated below;
  * one gray channel is gray_of, over all 2^24 triples;
  * the host-built tensor equals the restatement's conversion of the host-built RGBA crop, bit for bit, over the face
    crop corpus (golden CS boxes, random rotated boxes with NaN angles, scales 0.25 to 16, every orientation x mirror x
    source rectangle, every input format), in both layouts, three channel modes and four dtypes, with padded row and
    plane strides whose padding keeps its sentinel; records that keep no face write nothing;
  * the new bodies do not spill, k_face_crop stays at 64 registers, and the ABI exports the setter."""
import ctypes as C
import math
import re
import subprocess
from fractions import Fraction
from pathlib import Path

import numpy as np
import pytest

from headtrackr_b200 import _lib
from headtrackr_b200.context import tensor_affine
from test_cascade_host import CSRC, st  # noqa: F401  (fixture: the host-only build of ht_api.cu)
from test_face_crop_host import HALF_PI, event, golden_cs_boxes, lib_crop_rgba, lib_crop_yuv, smooth_frame
from test_formats_host import NEW, colors_of, fo, image, random_frame  # noqa: F401
from test_views_host import view_of

DTYPES = {"u8": _lib.HT_TENSOR_U8, "f16": _lib.HT_TENSOR_F16, "bf16": _lib.HT_TENSOR_BF16, "f32": _lib.HT_TENSOR_F32}
ESIZE = {"u8": 1, "f16": 2, "bf16": 2, "f32": 4}
NPTYPE = {"u8": np.uint8, "f16": np.uint16, "bf16": np.uint16, "f32": np.uint32}
LAYOUTS = {"chw": _lib.HT_TENSOR_CHW, "hwc": _lib.HT_TENSOR_HWC}
CHANNELS = {"rgb": _lib.HT_TENSOR_RGB, "bgr": _lib.HT_TENSOR_BGR, "gray": _lib.HT_TENSOR_GRAY}
IMAGENET_MEAN, IMAGENET_STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
SENTINEL = 0xA5


def _f32(x):
    return float(np.float32(x))


# (mul, add) pairs: ImageNet's three channels, plain 1/255, tiny, huge, f16- and bf16-overflowing, negative
AFFINE = [(_f32(1 / (255 * s)), _f32(-m / s)) for m, s in zip(IMAGENET_MEAN, IMAGENET_STD)] + [
    (_f32(1 / 255), 0.0), (1.0, 0.0), (_f32(1e-30), _f32(1e-38)), (_f32(3e-39), 0.0), (_f32(1e36), _f32(-1e35)),
    (300.0, -1000.5), (-300.0, 7.0), (2.0 ** 120, 2.0 ** 120 - 2.0 ** 104), (-2.0 ** 120, 2.0 ** 104 - 2.0 ** 120),
    (2.0 ** 120, 2.0 ** 127), (_f32(2.0 ** 120), _f32(-2.0 ** 127)), (_f32(1 / 3), _f32(-2 / 3)),
    (_f32(1e-3), _f32(65504.0)), (1.0, 65504.0)]


@pytest.fixture(scope="module")
def to(tmp_path_factory):
    """tests/crop_tensor_oracle.c built into a temporary directory, without contraction"""
    lib = tmp_path_factory.mktemp("crop_tensor_oracle") / "libcrop_tensor_oracle.so"
    subprocess.check_call(["cc", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", str(lib),
                           str(Path(__file__).with_name("crop_tensor_oracle.c")), "-lm"])
    L = C.CDLL(str(lib))
    L.hcto_values.argtypes = [C.c_int, C.c_float, C.c_float, C.c_void_p, C.c_longlong, C.c_void_p]
    L.hcto_values.restype = None
    L.hcto_gray.argtypes = [C.c_void_p, C.c_longlong, C.c_void_p]
    L.hcto_gray.restype = None
    L.hcto_convert.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                               C.c_void_p, C.c_longlong, C.c_longlong]
    L.hcto_convert.restype = None
    return L


@pytest.fixture(scope="module")
def lib(st):  # noqa: F811
    st.ht_selftest_face_crop.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    st.ht_selftest_face_crop_rgba.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    st.ht_selftest_face_tensor.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    st.ht_selftest_tensor_pixels.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    st.ht_selftest_tensor_pixels.restype = None
    return st


def record(data, w, h, dtype, layout, channels, mul, add, row, plane, scale=1.0):
    return _lib.FaceTensor(data, row, plane, w, h, DTYPES[dtype], LAYOUTS[layout], CHANNELS[channels], 0,
                           (C.c_float * 3)(*mul), (C.c_float * 3)(*add), scale)


# ---- the conversion ---------------------------------------------------------------------------------------------------

def lib_values(lib, dtype, mul, add, c):
    """the library's element bits for channel values c (as gray pixels through channel R of an HWC RGB row)"""
    px = (c.astype(np.uint32) * 0x010101 | 0xff000000).astype(np.uint32)
    out = np.zeros(3 * len(c), NPTYPE[dtype])
    t = record(out.ctypes.data, len(c), 1, dtype, "hwc", "rgb", [mul] * 3, [add] * 3, 3 * len(c), 0)
    lib.ht_selftest_tensor_pixels(C.addressof(t), px.ctypes.data, len(c))
    got = out.reshape(-1, 3)
    assert (got == got[:, :1]).all()
    return got[:, 0]


def oracle_values(to, dtype, mul, add, c):
    out = np.zeros(len(c), NPTYPE[dtype])
    cc = np.ascontiguousarray(c, np.uint8)
    to.hcto_values(DTYPES[dtype], mul, add, cc.ctypes.data, len(c), out.ctypes.data)
    return out


def exactly_rounded_f32(x):
    """the float32 nearest the rational x, ties to even (inf beyond the largest float's rounding boundary)"""
    big = Fraction(2) ** 128 - Fraction(2) ** 103            # halfway between FLT_MAX and 2^128
    if abs(x) >= big:
        return np.float32(math.copysign(math.inf, x))
    f = np.float32(float(x))                                   # within one ulp; then pick the nearest neighbour
    best = None
    with np.errstate(over="ignore"):
        near = (np.nextafter(f, np.float32(-np.inf)), f, np.nextafter(f, np.float32(np.inf)))
    for g in near:
        if not np.isfinite(g):
            continue
        d = abs(Fraction(float(g)) - x)
        even = (int(np.array(g).view(np.uint32)) & 1) == 0
        if best is None or d < best[0] or (d == best[0] and even):
            best = (d, g)
    return best[1]


def bf16_rne(f32_bits):
    u = f32_bits.astype(np.uint64)
    return ((u + 0x7fff + ((u >> 16) & 1)) >> 16).astype(np.uint16)


@pytest.mark.parametrize("dtype", ["f32", "f16", "bf16"])
def test_every_byte_every_affine(lib, to, dtype):
    c = np.arange(256, dtype=np.uint8)
    for mul, add in AFFINE:
        got = lib_values(lib, dtype, mul, add, c)
        assert np.array_equal(got, oracle_values(to, dtype, mul, add, c)), (dtype, mul, add)
        v32 = lib_values(lib, "f32", mul, add, c).view(np.float32)
        if dtype == "f32":
            for x in range(256):
                want = exactly_rounded_f32(Fraction(x) * Fraction(mul) + Fraction(add))
                assert v32[x] == want or (np.isinf(want) and v32[x] == want), (mul, add, x, v32[x], want)
        elif dtype == "f16":
            with np.errstate(over="ignore"):
                assert np.array_equal(got, v32.astype(np.float16).view(np.uint16)), (mul, add)
        else:
            assert np.array_equal(got, bf16_rne(v32.view(np.uint32))), (mul, add)


def test_overflow_gives_inf(lib):
    c = np.arange(256, dtype=np.uint8)
    f16 = lib_values(lib, "f16", 300.0, -1000.5, c)
    assert f16[255] == 0x7c00 and f16[0] == np.float16(-1000.5).view(np.uint16)
    assert lib_values(lib, "f16", -300.0, 7.0, c)[255] == 0xfc00
    top = 2.0 ** 120 - 2.0 ** 104                              # 255 x 2^120 + top is the largest float
    assert lib_values(lib, "f32", 2.0 ** 120, top, c).view(np.float32)[255] == np.finfo(np.float32).max
    assert lib_values(lib, "bf16", 2.0 ** 120, top, c)[255] == 0x7f80
    assert lib_values(lib, "bf16", -2.0 ** 120, -top, c)[255] == 0xff80
    f32 = lib_values(lib, "f32", 2.0 ** 120, 2.0 ** 127, c).view(np.float32)
    assert (f32[128:] == np.inf).all() and np.isfinite(f32[:128]).all()


def test_u8_is_the_byte(lib, to):
    c = np.arange(256, dtype=np.uint8)
    assert np.array_equal(lib_values(lib, "u8", 1.0, 0.0, c), c)
    assert np.array_equal(oracle_values(to, "u8", 1.0, 0.0, c), c)


def test_against_torchvision_two_step():
    """(x / 255 - mean) / std in fp32, two roundings per step, against fmaf(x, mul, add) with mul = f32(1 / (255 std)),
    add = f32(-mean / std): within 3 ulp of the larger of |v| and 1 / std (the cancellation near v = 0 is measured
    against the input scale), over every byte and ImageNet's three channels."""
    x = np.arange(256, dtype=np.float32)
    worst = 0.0
    for m, s in zip(IMAGENET_MEAN, IMAGENET_STD):
        two = (x / np.float32(255) - np.float32(m)) / np.float32(s)
        mul, add = _f32(1 / (255 * s)), _f32(-m / s)
        one = np.array([exactly_rounded_f32(Fraction(int(v)) * Fraction(mul) + Fraction(add)) for v in x], np.float32)
        scale = np.maximum(np.abs(two), np.float32(1 / s))
        ulp = np.spacing(scale.astype(np.float32))
        worst = max(worst, float((np.abs(one.astype(np.float64) - two.astype(np.float64)) / ulp).max()))
    assert worst <= 3.0, worst


def test_gray_is_gray_of_over_all_triples(lib, to):
    i = np.arange(1 << 24, dtype=np.uint32)
    px = i | np.uint32(0xff000000)
    want = np.empty(1 << 24, np.uint8)
    to.hcto_gray(px.ctypes.data, len(px), want.ctypes.data)
    got = np.zeros(1 << 24, np.uint8)
    t = record(got.ctypes.data, 1 << 24, 1, "u8", "chw", "gray", [1, 1, 1], [0, 0, 0], 1 << 24, 0)
    lib.ht_selftest_tensor_pixels(C.addressof(t), px.ctypes.data, len(px))
    assert np.array_equal(got, want)
    r, g, b = (i & 255).astype(np.float64), ((i >> 8) & 255).astype(np.float64), (i >> 16).astype(np.float64)
    assert np.array_equal(want, np.minimum(np.rint(r * 0.3 + g * 0.59 + b * 0.11), 255).astype(np.uint8))


# ---- tensors ----------------------------------------------------------------------------------------------------------

def tensor_layout(dtype, layout, channels, Sw, Sh, pad_row=0, pad_plane=0, lead=3):
    """(element offset of the tensor, row stride, plane stride, buffer elements) in one sentinel buffer"""
    n = 1 if channels == "gray" else 3
    if layout == "chw":
        row = Sw + pad_row
        plane = (Sh - 1) * row + Sw + pad_plane if n == 3 else 0
        size = (n - 1) * plane + (Sh - 1) * row + Sw
    else:
        row, plane = n * Sw + pad_row, 0
        size = (Sh - 1) * row + n * Sw
    return lead, row, plane, lead + size + 7


def affine_for(dtype, channels, seed=0):
    """(mul, add) of a test tensor: 1 and 0 for uint8, else ImageNet's (even seeds) or an arbitrary mix (odd seeds)"""
    if dtype == "u8":
        return [1.0] * 3, [0.0] * 3
    if seed % 2 == 0:
        n = 1 if channels == "gray" else 3
        mul = [_f32(1 / (255 * s)) for s in IMAGENET_STD[:n]] + [1.0] * (3 - n)
        add = [_f32(-m / s) for m, s in zip(IMAGENET_MEAN[:n], IMAGENET_STD[:n])] + [0.0] * (3 - n)
        return mul, add
    return [_f32(1 / 255), _f32(-2 / 255), 0.5], [-0.5, 1.0, _f32(1 / 3)]


def lib_tensor(lib, e, cw, ch, frame, dtype, layout, channels, mul, add, o=0, rect=(0, 0, 0, 0), Sw=24, Sh=20,
               scale=1.0, in_color=None, pad_row=0, pad_plane=0):
    """the host build's face tensor, of an RGBA8 frame (in_color None) or of a frame of any format -> (rc, buffer)"""
    lead, row, plane, size = tensor_layout(dtype, layout, channels, Sw, Sh, pad_row, pad_plane)
    buf = np.full(size * ESIZE[dtype], SENTINEL, np.uint8)
    t = record(buf.ctypes.data + lead * ESIZE[dtype], Sw, Sh, dtype, layout, channels, mul, add, row, plane, scale)
    view = view_of(o, rect)
    if in_color is None:
        h, w = frame.shape[:2]
        src = np.ascontiguousarray(frame)
        f = _lib.VideoFrame(src.ctypes.data, 0, w, h, 4 * w, 0.0)
        rc = lib.ht_selftest_face_tensor(C.addressof(e), cw, ch, None, C.addressof(f), C.addressof(view), C.addressof(t))
    else:
        img = image(frame, in_color)
        rc = lib.ht_selftest_face_tensor(C.addressof(e), cw, ch, C.addressof(img), None, C.addressof(view), C.addressof(t))
    return rc, buf


def convert_into(to, rgba_buf, rgba_pitch, dtype, layout, channels, mul, add, Sw, Sh, pad_row=0, pad_plane=0):
    """the restatement's conversion of an RGBA crop buffer into a sentinel buffer of tensor_layout"""
    lead, row, plane, size = tensor_layout(dtype, layout, channels, Sw, Sh, pad_row, pad_plane)
    buf = np.full(size * ESIZE[dtype], SENTINEL, np.uint8)
    to.hcto_convert(rgba_buf.ctypes.data, Sw, Sh, rgba_pitch, DTYPES[dtype], LAYOUTS[layout], CHANNELS[channels],
                    (C.c_float * 3)(*mul), (C.c_float * 3)(*add), buf.ctypes.data + lead * ESIZE[dtype], row, plane)
    return buf


def check(lib, to, e, cw, ch, frame, dtype, layout, channels, o=0, rect=(0, 0, 0, 0), Sw=24, Sh=20, scale=1.0, seed=0,
          **kw):
    """face tensor of an RGBA8 frame == the restatement's conversion of the RGBA crop; -> rc"""
    mul, add = affine_for(dtype, channels, seed)
    rc, got = lib_tensor(lib, e, cw, ch, frame, dtype, layout, channels, mul, add, o, rect, Sw, Sh, scale, **kw)
    a = lib_crop_rgba(lib, e, cw, ch, frame, o, rect, Sw, Sh, scale)
    assert rc == a[0], (e.x, e.y, e.width, e.height, e.angle, o, rect, Sw, Sh, scale)
    want = convert_into(to, a[1], a[2], dtype, layout, channels, mul, add, Sw, Sh, kw.get("pad_row", 0),
                        kw.get("pad_plane", 0))
    if not rc:
        want[:] = SENTINEL
    assert np.array_equal(got, want), (e.x, e.y, e.width, e.height, e.angle, o, rect, Sw, Sh, scale, dtype, layout, channels)
    return rc


MODES = [(d, l, c) for d in DTYPES for l in LAYOUTS for c in CHANNELS]


def test_golden_boxes(lib, to):
    frame = smooth_frame(160, 120, seed=4)
    made = 0
    for i, (x, y, w, h, a) in enumerate(golden_cs_boxes()):
        d, l, c = MODES[i % len(MODES)]
        made += check(lib, to, event(2, x, y, w, h, a), 160, 120, frame, d, l, c, Sw=28, Sh=24, scale=1.25, seed=i)
    assert made > 20


def test_random_rotated_boxes_scales_views(lib, to):
    rng = np.random.default_rng(29)
    frame = rng.integers(0, 256, (60, 80, 4), dtype=np.uint8)
    angles = [HALF_PI, math.nan, 0.0, -HALF_PI] + list(rng.uniform(-math.pi, math.pi, 6))
    scales = [0.25, 0.6, 1.0, 2.5, 16.0]
    sizes = [(24, 20), (1, 1), (48, 16), (11, 33)]
    n = 0
    for i, a in enumerate(angles):
        scale, (Sw, Sh) = scales[i % len(scales)], sizes[i % len(sizes)]
        e = event(2, float(rng.uniform(10, 150)), float(rng.uniform(10, 110)), float(rng.integers(4, 60)),
                  float(rng.integers(4, 60)), a)
        for o in range(8):
            W, H = (60, 80) if o & 1 else (80, 60)
            for rect in ((0, 0, 0, 0), (W // 5, H // 7, W - W // 3, H - H // 4)):
                d, l, c = MODES[(3 * i + o + (rect[2] > 0)) % len(MODES)]
                n += check(lib, to, e, 160, 120, frame, d, l, c, o, rect, Sw, Sh, scale, seed=i + o)
    assert n == len(angles) * 16


@pytest.mark.parametrize("dtype", list(DTYPES))
def test_every_layout_channel_mode_with_padding(lib, to, dtype):
    frame = smooth_frame(160, 120, seed=8)
    e = event(2, 70.0, 55.0, 40.0, 50.0, 1.1)
    for layout in LAYOUTS:
        for channels in CHANNELS:
            for pad_row, pad_plane in ((0, 0), (5, 0), (3, 17), (0, 9)):
                for seed in (0, 1):
                    assert check(lib, to, e, 160, 120, frame, dtype, layout, channels, Sw=30, Sh=26, seed=seed,
                                 pad_row=pad_row, pad_plane=pad_plane) == 1


@pytest.mark.parametrize("fmt_in", ["nv12", "i420"] + NEW)
def test_every_input_format(lib, to, fo, fmt_in):  # noqa: F811
    """a tensor of a frame of any format is the conversion of that frame's RGBA crop"""
    rng = np.random.default_rng(len(fmt_in) * 11 + 3)
    for k, color_in in enumerate(colors_of(fmt_in)):
        frame = random_frame(rng, fmt_in, 67, 45, offsets=(2, 6, 4) if fmt_in == "p010" else (1, 3, 2))
        for o, rect in ((0, (0, 0, 0, 0)), (5, (2, 1, 30, 60))):
            e = event(2, float(rng.uniform(10, 70)), float(rng.uniform(10, 50)), float(rng.integers(6, 40)),
                      float(rng.integers(6, 40)), float(rng.uniform(0, math.pi)))
            d, l, c = MODES[(5 * k + o) % len(MODES)]
            mul, add = affine_for(d, c, k)
            rc, got = lib_tensor(lib, e, 80, 60, frame, d, l, c, mul, add, o, rect, 22, 18, 1.2, in_color=color_in)
            a = lib_crop_yuv(lib, e, 80, 60, frame, color_in, o, rect, 22, 18, 1.2)
            assert rc == a[0] == 1
            assert np.array_equal(got, convert_into(to, a[1], a[2], d, l, c, mul, add, 22, 18)), (fmt_in, color_in, o)


def test_pixels_outside_the_video_are_add(lib, to):
    frame = np.full((120, 160, 4), 200, np.uint8)
    e = event(2, -30.0, -30.0, 40.0, 40.0, HALF_PI)
    mul, add = [_f32(1 / 255)] * 3, [-0.25, 0.5, 2.0]
    rc, got = lib_tensor(lib, e, 160, 120, frame, "f32", "chw", "rgb", mul, add, Sw=16, Sh=16)
    assert rc == 1 and check(lib, to, e, 160, 120, frame, "f32", "chw", "rgb", Sw=16, Sh=16)
    v = got[3 * 4:3 * 4 + 4 * 16 * 16 * 3].view(np.float32).reshape(3, 16, 16)
    assert v[0, 0, 0] == np.float32(-0.25) and v[1, 0, 0] == np.float32(0.5) and v[2, 0, 0] == np.float32(2.0)


def test_records_that_keep_no_face_write_nothing(lib):
    frame = smooth_frame(160, 120)
    for e in (event(1, 50, 50, 30, 30, 0.0), event(2, 50, 50, 0, 30, HALF_PI), event(2, math.nan, 50, 30, 30, HALF_PI),
              event(0, 50, 50, 30, 30, 0.0)):
        for d, l, c in MODES[::5]:
            mul, add = affine_for(d, c, 1)
            rc, got = lib_tensor(lib, e, 160, 120, frame, d, l, c, mul, add, Sw=16, Sh=16)
            assert rc == 0 and (got == SENTINEL).all()


# ---- the kernel and the ABI -------------------------------------------------------------------------------------------

def test_tensor_bodies_do_not_spill_and_k_face_crop_keeps_64_registers(tmp_path):
    out = subprocess.run([_lib.nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-fmad=false",
                          "-Xptxas", "-v", "-Xcompiler", "-fPIC", "-c", "-o", str(tmp_path / "ht_api.o"),
                          str(CSRC / "ht_api.cu")], capture_output=True, text=True, check=True).stderr
    names = ["k_face_crop"] + [f"face_tensor_tileILi{k}E" for k in range(3)]
    for name in names:
        m = re.search(r"Function properties for \S*" + name + r"\S*\n\s*(\d+) bytes stack frame, (\d+) bytes spill "
                      r"stores, (\d+) bytes spill loads", out)
        assert m, (name, out[-2000:])
        assert m.group(2) == m.group(3) == "0", m.group(0)
    m = re.search(r"Compiling entry function '\S*k_face_crop\S*' for 'sm_90a'\n(?:.*\n)*?ptxas info\s*: Used (\d+) "
                  r"registers", out)
    assert m and int(m.group(1)) <= 64, m and m.group(0)


def test_abi():
    L = _lib.lib()
    assert hasattr(L, "ht_tracker_set_face_tensor") and "ht_tracker_set_face_tensor" in _lib.EXPORTS
    assert L.ht_tracker_set_face_tensor(None, 0, 1, (_lib.FaceTensor * 1)()) == _lib.HT_ERR_ARG
    header = (CSRC.parent.parent / "include" / "headtrackr_b200.h").read_text()
    assert "int ht_tracker_set_face_tensor(ht_ctx *ctx, int first, int n, const ht_face_tensor *tensors);" in header
    assert "} ht_face_tensor;         /* 80 bytes */" in header
    offs = {f: getattr(_lib.FaceTensor, f).offset for f in ("data", "row_stride", "plane_stride", "width", "height",
                                                            "dtype", "layout", "channels", "pad_", "mul", "add", "scale")}
    assert offs == dict(data=0, row_stride=8, plane_stride=16, width=24, height=28, dtype=32, layout=36, channels=40,
                        pad_=44, mul=48, add=60, scale=72)
    for name, v in (("U8", 0), ("F16", 1), ("BF16", 2), ("F32", 3), ("CHW", 0), ("HWC", 1), ("RGB", 0), ("BGR", 1),
                    ("GRAY", 2)):
        assert f"#define HT_TENSOR_{name} {v}\n" in header and getattr(_lib, f"HT_TENSOR_{name}") == v


def test_tensor_affine_rounds_once_from_float64():
    import torch
    mul, add = tensor_affine(torch.float16, "rgb", IMAGENET_MEAN, IMAGENET_STD)
    for k in range(3):
        assert mul[k] == float(np.float32(1.0 / (255.0 * IMAGENET_STD[k])))
        assert add[k] == float(np.float32(-IMAGENET_MEAN[k] / IMAGENET_STD[k]))
    assert tensor_affine(torch.uint8, "gray") == ([1.0] * 3, [0.0] * 3)
    mul, add = tensor_affine(torch.float32, "gray", 0.5, 0.25)           # gray uses channel 0 only
    assert (mul[0], add[0]) == (_f32(1 / 63.75), -2.0)
    with pytest.raises(ValueError):
        tensor_affine(torch.uint8, "rgb", IMAGENET_MEAN, IMAGENET_STD)
    with pytest.raises(ValueError):
        tensor_affine(torch.float16, "rgb", (0.5, 0.5), 1.0)
