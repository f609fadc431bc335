"""CPU: the video draw of ht_tracker_feed (drawImage(video, 0, 0, canvas.width, canvas.height), src/main.js:170,312,
once per listed stream, each with its own video size and row pitch) - k_feed_draw's per-record code run on the host
over a heterogeneous record batch against the oracle's canvas-shim drawImage; the replication identity the GPU replay
of the goldens through ht_tracker_feed relies on; and the ABI of the new entry point."""
import ctypes as C

import numpy as np
import pytest

import oracle
from headtrackr_b200 import _lib, synth
from test_cascade_host import st  # noqa: F401  (fixture: the host-only build of ht_api.cu)
from test_host_lifecycle import GOLD_L, make_frame


def oracle_resize(frame, dw, dh):
    sh, sw = frame.shape[:2]
    out = np.zeros((dh, dw, 4), np.uint8)
    for c in range(4):
        out[..., c] = oracle.draw_image(np.ascontiguousarray(frame[..., c]), 0, 0, sw, sh, dw, dh, dw, dh)
    return out


def padded(frame, extra_px, fill=0xAB):
    """a row-padded view of `frame`: rows of (w + extra_px) pixels, the padding filled with `fill`"""
    h, w = frame.shape[:2]
    buf = np.full((h, w + extra_px, 4), fill, np.uint8)
    buf[:, :w] = frame
    return buf[:, :w]


def feed_draw(st, videos, draw, dw, dh, canvas):
    st.ht_selftest_feed_draw.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    recs = (_lib.VideoFrame * len(videos))()
    for b, v in enumerate(videos):
        assert v.strides[1:] == (4, 1)
        recs[b] = _lib.VideoFrame(v.ctypes.data, b, v.shape[1], v.shape[0], v.strides[0], 0.0)
    d = np.asarray(draw, np.uint8)
    assert st.ht_selftest_feed_draw(C.addressof(recs), len(videos), d.ctypes.data, canvas.ctypes.data, dw, dh) == 0


def test_heterogeneous_record_batch_equals_the_oracle(st):
    dw, dh = 320, 240
    sizes = [(640, 480), (333, 251), (160, 120), (1280, 720), (200, 150)]
    videos = [synth.frame(90 + i, w, h) for i, (w, h) in enumerate(sizes)]
    videos[1][..., 3] = (np.arange(sizes[1][0]) % 256).astype(np.uint8)[None, :]   # a non-constant alpha channel too
    videos[1] = padded(videos[1], 13)                                                 # pitch = 4 * 346 > 4 * 333
    assert videos[1].strides[0] == 4 * 346
    draw = [1, 1, 1, 1, 0]                                                            # the last stream is IDLE
    canvas = np.random.default_rng(5).integers(0, 256, (len(videos), dh, dw, 4), dtype=np.uint8)
    before = canvas.copy()
    feed_draw(st, videos, draw, dw, dh, canvas)
    for b, v in enumerate(videos):
        if draw[b]:
            assert np.array_equal(canvas[b], oracle_resize(np.ascontiguousarray(v), dw, dh)), sizes[b]
        else:
            assert np.array_equal(canvas[b], before[b])


def test_one_to_one_record_is_a_copy(st):
    v = padded(synth.frame(3, 160, 120), 4)
    canvas = np.zeros((1, 120, 160, 4), np.uint8)
    feed_draw(st, [v], [1], 160, 120, canvas)
    assert np.array_equal(canvas[0], v)
    assert np.array_equal(oracle_resize(np.ascontiguousarray(v), 160, 120), v)


@pytest.mark.parametrize("k", [1, 2, 3, 4])
def test_replicated_golden_frame_draws_back_exactly(st, k):
    """A golden frame replicated k x k per pixel draws back onto the golden's canvas exactly: every bilinear tap of
    canvas pixel (X, Y) falls inside the k x k block of (X, Y).  So a stream fed its golden at k times the size must
    replay the golden bit for bit."""
    W, H = GOLD_L["width"], GOLD_L["height"]
    for kind, t in (("face", 3), ("ramp", 2), ("empty", 0)):
        f = make_frame(kind, t)
        big = np.ascontiguousarray(np.repeat(np.repeat(f, k, axis=0), k, axis=1))
        assert np.array_equal(oracle_resize(big, W, H), f), (kind, k)
        canvas = np.zeros((1, H, W, 4), np.uint8)
        feed_draw(st, [big], [1], W, H, canvas)
        assert np.array_equal(canvas[0], f), (kind, k)


def test_tracker_feed_abi():
    L = _lib.lib()
    assert hasattr(L, "ht_tracker_feed") and "ht_tracker_feed" in _lib.EXPORTS
    assert C.sizeof(_lib.VideoFrame) == 32
    assert (_lib.VideoFrame.stream.offset, _lib.VideoFrame.width.offset, _lib.VideoFrame.height.offset,
            _lib.VideoFrame.pitch.offset, _lib.VideoFrame.now_ms.offset) == (8, 12, 16, 20, 24)
    v = L.ht_version()
    assert v >> 16 == 1 and (v & 0xffff) >= 2
