"""CPU: where pipelined ht_detect_track calls put their bin planes and histograms (ht_set_pipeline, DESIGN.md §5.5).

The tracking of pipelined call s still reads its bin planes and current-frame histograms while the gray pass of call
s+1 writes its own; nothing orders the two.  So the slices of two consecutive pipelined calls must not share a byte,
whatever frame size and batch size each call has, unless a synchronisation separates them: the bin-plane buffer grows
only behind one, and every other entry point joins the pending tracking and starts the parities over.  Every slice is
16-byte aligned: k_gray's 8-byte plane stores, k_bins_mask's 16-byte groups and k_track's 8-byte plane loads then only
depend on the frame size (w % 4 == 0 makes every frame's plane start 8-byte aligned).

ht_selftest_pipe_offsets returns what pipe_plane_offsets, the rule the pipelined call uses, gives; here the calls of a
sequence are replayed through it, with the buffer's growth (DevBuf::reserve only grows) and the joins restated from the
library.
"""
import ctypes as C
import random

import pytest

from test_cascade_host import st  # noqa: F401  (fixture: the host-only build of ht_api.cu)

A, B, C_, ODD1, ODD2 = (320, 240), (160, 120), (256, 192), (161, 121), (97, 83)
JOIN = "join"      # a call of any other entry point (or one with host outputs): joins, then uses parity 0


@pytest.fixture(scope="module")
def po(st):
    st.ht_selftest_pipe_offsets.argtypes = [C.c_int, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_void_p]
    st.ht_selftest_pipe_offsets.restype = None
    return st


def slices(po, parity, cap, max_frames, w, h):
    out = (C.c_uint64 * 3)()
    po.ht_selftest_pipe_offsets(parity, cap, max_frames, w, h, out)
    return tuple(out)


def replay(po, max_frames, calls):
    """calls: [(w, h, n) of a pipelined call, or (JOIN, w, h, n) of a joining call with n x w x h frames].
    -> [what is wrong], each with the byte ranges involved"""
    cap, parity, prev, bad = 0, 0, None, []
    hist_bytes = 2 * max_frames * 4096 * 4                    # ensure_tracker_buffers: two parities
    for i, call in enumerate(calls):
        if call[0] == JOIN:
            _, w, h, n = call
            cap = max(cap, 2 * n * w * h)                     # the unpipelined call's reserve (n frames' planes)
            parity, prev = 0, None
            continue
        w, h, n = call
        parity ^= 1
        grow, boff, hoff = slices(po, parity, cap, max_frames, w, h)
        if grow:
            assert grow > cap
            cap, prev = grow, None                            # both streams are synchronised before the buffer moves
        bins = (2 * boff, 2 * (boff + n * w * h))
        hist = (4 * hoff, 4 * (hoff + n * 4096))
        tag = f"call {i} ({w}x{h}, n={n}, parity {parity})"
        if bins[1] > cap or hist[1] > hist_bytes:
            bad.append(f"{tag}: bins {bins} / hist {hist} outside the buffers ({cap}, {hist_bytes} bytes)")
        if bins[0] % 16 or hist[0] % 16:
            bad.append(f"{tag}: bins at byte {bins[0]}, hist at byte {hist[0]}: not 16-byte aligned")
        if prev is not None:
            for name, now, before in (("bins", bins, prev[1]), ("hist", hist, prev[2])):
                if now[0] < before[1] and before[0] < now[1]:
                    bad.append(f"{tag} writes {name} bytes {now} while {prev[0]} still reads {before}")
        prev = (tag, bins, hist)
    return bad


def piped(*sizes, n):
    return [(w, h, n) for w, h in sizes]


# the sequences tests/test_gpu_pipeline_shapes.py runs on the device
SEQUENCES = {
    "worked example A A B": (12, piped(A, A, B, n=12)),
    "sizes both ways": (12, piped(A, A, B, B, A, B, A, A, n=12)),
    "batch sizes and a third size": (12, [(*A, 12), (*C_, 7), (*B, 1), (*A, 12), (*C_, 12), (*B, 7), (*A, 12)]),
    "odd plane sizes": (13, [(*ODD1, 13), (*ODD2, 13), (*ODD1, 5), (*ODD2, 13), (*ODD1, 13), (*ODD2, 1)]),
    "one size (interval changes)": (12, piped(A, A, A, n=12)),
    "a joining call in the middle": (12, piped(A, A, n=12) + [(JOIN, *A, 12)] + piped(B, B, A, n=12)),
    "tiers": (192, piped((160, 120), (160, 120), (128, 96), (128, 96), (160, 120), n=192)),
    "small after a grown buffer": (12, piped(B, A, B, A, n=12)),
}


@pytest.mark.parametrize("name", list(SEQUENCES))
def test_device_sequences(po, name):
    max_frames, calls = SEQUENCES[name]
    bad = replay(po, max_frames, calls)
    assert not bad, "\n".join(bad)


def test_random_sequences(po):
    sizes = [A, B, C_, ODD1, ODD2, (640, 480), (24, 24), (25, 24), (33, 31), (1280, 720), (128, 96), (333, 251)]
    rng = random.Random(90)
    for trial in range(600):
        max_frames = rng.choice([1, 2, 3, 4, 5, 7, 12, 13, 64, 192, 1024])
        calls = []
        for _ in range(rng.randint(2, 14)):
            w, h = rng.choice(sizes)
            n = rng.choice([1, max_frames, rng.randint(1, max_frames)])
            calls.append((JOIN, w, h, n) if rng.random() < 0.1 else (w, h, n))
        bad = replay(po, max_frames, calls)
        assert not bad, (trial, max_frames, calls, bad)


@pytest.mark.parametrize("max_frames,w,h", [(1024, 640, 480), (12, 320, 240), (192, 160, 120), (512, 1280, 720)])
def test_fixed_size_keeps_the_plain_parity_offsets(po, max_frames, w, h):
    """One frame size with max_frames * w * h a multiple of 8 (every bench configuration): the slices are parity times
    one parity's planes, as for a buffer of exactly two parities."""
    plane = max_frames * w * h
    assert plane % 8 == 0
    cap = 0
    for call in range(6):
        parity = (call + 1) & 1
        grow, boff, hoff = slices(po, parity, cap, max_frames, w, h)
        assert grow == (4 * plane if call == 0 else 0)
        cap = max(cap, grow)
        assert (boff, hoff) == (parity * plane, parity * max_frames * 4096)
