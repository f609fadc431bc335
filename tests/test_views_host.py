"""CPU: views of video frames (DESIGN.md 2, "Views"): an orientation and a source rectangle applied by the canvas draw.

  * the orientation formulas equal numpy's rot90 / fliplr on odd, even, 1xN and Nx1 frames (k_feed_draw_view's
    per-record code, compiled for the host, drawing 1:1), and the EXIF and rotation + flip tags map onto them;
  * the draw (ht_selftest_feed_view) equals hto_draw_image over the numpy-oriented frame of format_oracle's RGBA8
    frame, per channel, for every orientation, format and colour, crops of every kind, 1:1, down- and up-scaled, with
    planes on and off 2- and 4-byte boundaries, and through the upright and the transposed thread layout alike;
  * every bad view is rejected;
  * headtrackr_b200.views maps canvas points, boxes and tracked objects back to the video as brute force does;
  * the ABI, and a spill-free k_feed_draw_view."""
import ctypes as C
import math
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest

import oracle
from headtrackr_b200 import _lib, views
from test_cascade_host import CSRC, st  # noqa: F401  (fixture: the host-only build of ht_api.cu)
from test_formats_host import NEW, RGB, YUV_COLORS, fo, image, oracle_convert, random_frame  # noqa: F401

ALL = ["nv12", "i420"] + NEW


def orient_np(a, o):
    """the oriented frame of an (h, w, ...) array: rotate clockwise by 90 * (o & 3), then mirror if o & 4"""
    r = np.rot90(a, -(o & 3))
    return np.ascontiguousarray(np.fliplr(r) if o & 4 else r)


def view_of(o, crop=(0, 0, 0, 0), reserved=(0, 0, 0)):
    return _lib.VideoView(o, *crop, (C.c_int32 * 3)(*reserved))


def draw_rgba(st, rgba, view, dw, dh, pitch_extra=0):
    st.ht_selftest_feed_view_rgba.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    h, w = rgba.shape[:2]
    buf = np.zeros((h, w + pitch_extra, 4), np.uint8)
    buf[:, :w] = rgba
    f = _lib.VideoFrame(buf.ctypes.data, 0, w, h, 4 * (w + pitch_extra), 0.0)
    canvas = np.zeros((dh, dw, 4), np.uint8)
    rc = st.ht_selftest_feed_view_rgba(C.addressof(f), C.addressof(view), canvas.ctypes.data, dw, dh)
    return rc, canvas


def draw_yuv(st, frame, color, view, dw, dh):
    st.ht_selftest_feed_view.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    img = image(frame, color)
    canvas = np.zeros((dh, dw, 4), np.uint8)
    rc = st.ht_selftest_feed_view(C.addressof(img), C.addressof(view), canvas.ctypes.data, dw, dh)
    return rc, canvas


def oracle_view(rgba, o, crop, dw, dh):
    """hto_draw_image(orient(rgba), sx, sy, sw, sh, 0, 0, dw, dh), channel by channel"""
    O = orient_np(rgba, o)
    sx, sy, sw, sh = crop if any(crop) else (0, 0, O.shape[1], O.shape[0])
    out = np.zeros((dh, dw, 4), np.uint8)
    for c in range(4):
        out[..., c] = oracle.draw_image(np.ascontiguousarray(O[..., c]), sx, sy, sw, sh, dw, dh, dw, dh)
    return out


# ---- 1. the orientation formulas ------------------------------------------------------------------------------------

SHAPES = [(1, 1), (7, 5), (8, 6), (1, 9), (9, 1), (33, 17)]       # (w, h)


@pytest.mark.parametrize("size", SHAPES, ids=[f"{w}x{h}" for w, h in SHAPES])
def test_orientations_equal_numpy(st, size):
    w, h = size
    rng = np.random.default_rng(w * 31 + h)
    V = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    for o in range(8):
        O = orient_np(V, o)
        assert views.oriented_size({"rotate": 90 * (o & 3)}, w, h) == (O.shape[1], O.shape[0])
        rc, got = draw_rgba(st, V, view_of(o), O.shape[1], O.shape[0], pitch_extra=o % 3)
        assert rc == 0 and np.array_equal(got, O), (size, o)
        # the table of include/headtrackr_b200.h, pixel by pixel
        W = O.shape[1]
        for y in range(O.shape[0]):
            for x in range(W):
                xm = W - 1 - x if o & 4 else x
                vx, vy = [(xm, y), (y, h - 1 - xm), (w - 1 - xm, h - 1 - y), (w - 1 - y, xm)][o & 3]
                assert np.array_equal(O[y, x], V[vy, vx])


def exif_np(a, tag):
    """the upright image of a stored (h, w, ...) image with EXIF orientation `tag`, by the tag's definition"""
    return {1: lambda: a, 2: lambda: a[:, ::-1], 3: lambda: a[::-1, ::-1], 4: lambda: a[::-1],
            5: lambda: a.transpose(1, 0, 2), 6: lambda: np.rot90(a, -1), 7: lambda: a[::-1, ::-1].transpose(1, 0, 2),
            8: lambda: np.rot90(a, 1)}[tag]()


def test_exif_and_rotation_flip_tags(st):
    V = np.arange(5 * 3 * 4, dtype=np.uint8).reshape(3, 5, 4)          # asymmetric: every pixel distinct
    assert views.EXIF_ORIENTATION == {1: 0, 2: 4, 3: 2, 4: 6, 5: 5, 6: 1, 7: 7, 8: 3}
    for tag in range(1, 9):
        want = exif_np(V, tag)
        v = views.from_exif(tag)
        assert views.orientation(v) == views.EXIF_ORIENTATION[tag]
        rc, got = draw_rgba(st, V, views.video_view(v), want.shape[1], want.shape[0])
        assert rc == 0 and np.array_equal(got, want), tag
    for rotate in (0, 90, 180, 270):
        for flip in (False, True):
            want = np.rot90(V, -rotate // 90)
            want = want[:, ::-1] if flip else want
            rc, got = draw_rgba(st, V, views.video_view(views.from_tag(rotate, flip)), want.shape[1], want.shape[0])
            assert rc == 0 and np.array_equal(got, want), (rotate, flip)


# ---- 2. the draw against the oracle ---------------------------------------------------------------------------------

def crops(W, H):
    """whole frame, interior, touching each edge, 1x1, 1-pixel strips"""
    out = [(0, 0, 0, 0), (0, 0, W, H), (1, 1, max(1, W - 3), max(1, H - 2)), (0, 0, 1, 1), (W - 1, H - 1, 1, 1),
           (0, 0, W, 1), (0, H - 1, W, 1), (0, 0, 1, H), (W - 1, 0, 1, H), (W // 2, 0, W - W // 2, H // 2 + 1),
           (0, H // 3, W // 2 + 1, H - H // 3)]
    return [c for c in out if c[0] + c[2] <= W and c[1] + c[3] <= H and (not any(c) or min(c[2], c[3]) >= 1)]


def canvases(crop, W, H):
    """1:1, down-scaled and up-scaled canvases of a crop (the thread layout does not matter on the host; on the
    device both layouts draw the same canvases, tests/test_gpu_views.py)"""
    sw, sh = (crop[2], crop[3]) if any(crop) else (W, H)
    return [(sw, sh), (max(1, sw // 2), max(1, (2 * sh) // 3)), (2 * sw + 1, sh + 3)]


@pytest.mark.parametrize("fmt", ALL)
def test_draw_is_the_resampler_over_the_oriented_oracle_frame(st, fo, fmt):
    rng = np.random.default_rng(len(fmt) * 977)
    colors = ["bt601"] if fmt in RGB else YUV_COLORS
    n = 0
    for k, (w, h) in enumerate([(13, 9), (16, 10)]):
        # planes on 4-byte boundaries and off them by 1 and 2 (P010: by 2 and 4)
        for j, off in enumerate((0, 2, 4) if fmt == "p010" else (0, 1, 2)):
            color = colors[(k + j) % len(colors)]
            f = random_frame(rng, fmt, w, h, (off,) * 3, (j, 2 * j, j) if fmt != "p010" else (2 * j,) * 3)
            rgba = oracle_convert(fo, f, color)
            for o in range(8):
                W, H = (h, w) if o & 1 else (w, h)
                for crop in crops(W, H)[(o + j) % 2::2] if j else crops(W, H):
                    for dw, dh in canvases(crop, W, H):
                        rc, got = draw_yuv(st, f, color, view_of(o, crop), dw, dh)
                        assert rc == 0
                        assert np.array_equal(got, oracle_view(rgba, o, crop, dw, dh)), (fmt, color, w, o, crop, dw, dh)
                        n += 1
    assert n > 300


@pytest.mark.parametrize("size", [(64, 48), (41, 23)], ids=["64x48", "41x23"])
def test_rgba_draw_is_the_resampler_over_the_oriented_frame(st, size):
    w, h = size
    rng = np.random.default_rng(w)
    V = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    for o in range(8):
        W, H = (h, w) if o & 1 else (w, h)
        for crop in crops(W, H):
            for dw, dh in canvases(crop, W, H) + [(W // 4 + 1, H // 4 + 1)]:
                rc, got = draw_rgba(st, V, view_of(o, crop), dw, dh, pitch_extra=o)
                assert rc == 0 and np.array_equal(got, oracle_view(V, o, crop, dw, dh)), (o, crop, dw, dh)


def test_identity_view_equals_the_plain_draw(st, fo):
    """o = 0 over the whole frame is the draw of ht_selftest_feed_yuv"""
    from test_formats_host import selftest_draw
    rng = np.random.default_rng(3)
    for fmt in ALL:
        color = "bt601" if fmt in RGB else "bt709"
        f = random_frame(rng, fmt, 37, 21)
        for dw, dh in ((37, 21), (20, 12), (60, 40)):
            rc, got = draw_yuv(st, f, color, view_of(0), dw, dh)
            assert rc == 0 and np.array_equal(got, selftest_draw(st, f, color, dw, dh)), (fmt, dw)


# ---- 3. rejections --------------------------------------------------------------------------------------------------

def test_bad_views_are_rejected(st):
    rng = np.random.default_rng(9)
    V = rng.integers(0, 256, (6, 10, 4), dtype=np.uint8)              # 10 x 6; oriented 6 x 10 for 90 / 270
    f = random_frame(rng, "nv12", 10, 6)
    bad = [view_of(8), view_of(-1), view_of(0, reserved=(1, 0, 0)), view_of(0, reserved=(0, 0, -1)),
           view_of(0, (0, 0, 0, 1)), view_of(0, (0, 0, 1, 0)), view_of(0, (-1, 0, 2, 2)), view_of(0, (0, -1, 2, 2)),
           view_of(0, (9, 0, 2, 1)), view_of(0, (0, 5, 1, 2)), view_of(0, (0, 0, 11, 1)), view_of(1, (0, 0, 7, 1)),
           view_of(3, (0, 0, 1, 11)), view_of(5, (0, 9, 1, 2)), view_of(0, (1, 0, 0, 0)), view_of(2, (0, 0, -3, 2)),
           view_of(0, (0, 0, 2**31 - 1, 1)), view_of(0, (5, 0, 2**31 - 1, 1))]
    for i, v in enumerate(bad):
        rc, canvas = draw_rgba(st, V, v, 8, 8)
        assert rc == _lib.HT_ERR_ARG and not canvas.any(), i
        rc, canvas = draw_yuv(st, f, "bt601", v, 8, 8)
        assert rc == _lib.HT_ERR_ARG and not canvas.any(), i
    for good in (view_of(1, (0, 0, 6, 10)), view_of(7, (5, 9, 1, 1)), view_of(4, (9, 5, 1, 1))):
        assert draw_rgba(st, V, good, 8, 8)[0] == 0
    with pytest.raises(ValueError):
        views.video_view({"rotate": 45})
    with pytest.raises(ValueError):
        views.video_view({"crop": (0, 0, 0, 4)})


# ---- 4. canvas -> video ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("o", range(8))
def test_canvas_to_video_against_brute_force(o):
    w, h = 23, 14
    idx = np.stack(np.meshgrid(np.arange(w), np.arange(h)), -1)       # idx[y, x] = (x, y) of the video
    O = orient_np(idx, o)
    W, H = O.shape[1], O.shape[0]
    view = {"rotate": 90 * (o & 3), "mirror": bool(o & 4)}
    for crop in [None, (2, 3, W - 5, H - 4), (W - 3, 0, 3, H)]:
        v = dict(view, crop=crop)
        sx, sy, sw, sh = crop or (0, 0, W, H)
        for cw, ch in ((sw, sh), (2 * sw, 3 * sh)):                   # 1:1, and each crop pixel a 2x3 block
            kx, ky = cw // sw, ch // sh
            for Y in range(0, ch, 2):
                for X in range(0, cw, 3):
                    # the canvas pixel's centre lies in crop pixel (X // kx, Y // ky): its video pixel holds it
                    vx, vy = views.to_video(v, w, h, cw, ch, X + 0.5, Y + 0.5)
                    assert (math.floor(vx), math.floor(vy)) == tuple(O[sy + Y // ky, sx + X // kx]), (o, crop, X, Y)
            # a box of whole crop pixels covers exactly the video pixels those hold
            bx, by, bw, bh = views.box_to_video(v, w, h, cw, ch, kx, ky, 2 * kx, 3 * ky)
            cover = O[sy + 1:sy + 4, sx + 1:sx + 3].reshape(-1, 2)
            assert (bx, by) == (cover[:, 0].min(), cover[:, 1].min()), (o, crop)
            assert (bw, bh) == (cover[:, 0].max() + 1 - bx, cover[:, 1].max() + 1 - by), (o, crop)


def test_tracked_object_to_video():
    w, h = 40, 30
    for o in range(8):
        v = {"rotate": 90 * (o & 3), "mirror": bool(o & 4), "crop": None}
        W, H = views.oriented_size(v, w, h)
        for angle in (math.pi / 2, 0.3, 2.0):
            cx, cy, vw, vh, a = views.cs_to_video(v, w, h, W, H, 10.0, 12.0, 6.0, 9.0, angle)
            assert (cx, cy) == views.to_video(v, w, h, W, H, 10.0, 12.0)
            assert (vw, vh) == pytest.approx((6.0, 9.0))               # 1:1: the sizes stay
            # the height axis' end maps to the video along the returned angle
            ex, ey = views.to_video(v, w, h, W, H, 10.0 + math.cos(angle), 12.0 + math.sin(angle))
            d = math.atan2(ey - cy, ex - cx) % math.pi
            assert a == pytest.approx(d % math.pi, abs=1e-12) or abs(abs(a - d) - math.pi) < 1e-12, (o, angle)
            want = {0: angle, 2: angle, 4: math.pi - angle, 6: math.pi - angle}.get(o)
            if want is not None:                                       # upright views keep the angle, mirrors negate it
                assert a == pytest.approx(want % math.pi)
        # an upright object (angle pi/2) of a 90 / 270 view lies along the video's rows
        if o & 1:
            assert views.cs_to_video(v, w, h, W, H, 5.0, 5.0, 4.0, 8.0, math.pi / 2)[4] == pytest.approx(0.0, abs=1e-12)
    # scaled: a 2x canvas halves the sizes
    v = {"rotate": 90, "crop": (0, 0, 30, 40)}
    assert views.cs_to_video(v, w, h, 60, 80, 10.0, 10.0, 6.0, 8.0, math.pi / 2)[2:4] == pytest.approx((3.0, 4.0))


# ---- 5. ABI and registers -------------------------------------------------------------------------------------------

def test_views_abi():
    assert C.sizeof(_lib.VideoView) == 32
    assert [_lib.VideoView.orientation.offset, _lib.VideoView.sx.offset, _lib.VideoView.sy.offset, _lib.VideoView.sw.offset,
            _lib.VideoView.sh.offset, _lib.VideoView.reserved.offset] == [0, 4, 8, 12, 16, 20]
    header = (Path(__file__).resolve().parent.parent / "include" / "headtrackr_b200.h").read_text()
    for name, value in (("ROTATE_90", 1), ("ROTATE_180", 2), ("ROTATE_270", 3), ("MIRROR", 4)):
        assert re.search(rf"#define HT_VIEW_{name} {value}\b", header), name
        assert getattr(_lib, f"HT_VIEW_{name}") == value
    L = _lib.lib()
    for name in ("ht_tracker_feed_views", "ht_tracker_feed_yuv_views", "ht_ingest_views", "ht_ingest_yuv_views"):
        assert hasattr(L, name) and name in _lib.EXPORTS
    assert L.ht_version() == (1 << 16) | 3


def test_feed_draw_view_does_not_spill(tmp_path):
    """ptxas -v of the library as build() compiles it: k_feed_draw_view and its out-of-line CTA per texel source keep
    everything in registers"""
    out = subprocess.run([_lib.nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-fmad=false",
                          "-Xptxas", "-v", "-Xcompiler", "-fPIC", "-c", "-o", str(tmp_path / "ht_api.o"),
                          str(CSRC / "ht_api.cu")], capture_output=True, text=True, check=True).stderr
    found = re.findall(r"Function properties for (\S*feed_draw_view\S*)\n\s*(\d+) bytes stack frame, (\d+) bytes spill "
                       r"stores, (\d+) bytes spill loads", out)
    assert len(found) == 4, out[-2000:]                                # the kernel and its three CTA functions
    for name, _, stores, loads in found:
        assert (stores, loads) == ("0", "0"), name
