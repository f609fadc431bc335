"""CPU: the detector across canvas geometries, from the smallest frame the reference accepts to the planner's size limit.

Three checks, none of which needs a GPU:

- accept/reject: over a grid of small frames, the planner (build_plan, through ht_selftest_planes) accepts a frame
  exactly when the oracle's detect_objects (src/ccv.js:110-147) runs on it, and then plans the oracle's slot sizes;
- the large boundary: every limit of build_plan restated from the arithmetic it protects (the resample jobs of
  src/ccv.js:117-145, their 16-bit tap indices and the 32-bit division of k_resample) - the planner must accept a frame
  exactly when all of them hold, along the 16:9 line and along fixed-height and fixed-width lines, at every interval;
- emulation: every geometry of GEOMETRIES through k_gray's and k_resample's per-thread code and k_cascade's tile code
  (test_pyramid_host.py, test_cascade_host.py) against the oracle's pyramid planes and raw detection lists.

GEOMETRIES is shared with tests/test_gpu_detect_geometry.py, which runs the same frames through the CUDA kernels.
"""
import ctypes as C
import math

import numpy as np
import pytest

import oracle
from headtrackr_b200 import synth
from test_cascade_host import st, want_raw  # noqa: F401  (fixture + helper)
from test_pyramid_host import host_arena

INTERVALS = (1, 2, 3, 5)

# (W, H, intervals the frame is run at, the edge it exercises).  Every entry is accepted at each of its intervals.
GEOMETRIES = [
    (64, 64, (1, 2), "smallest frame at intervals 1 and 2: the last slot is 1 pixel wide, most scales have qw <= 0"),
    (77, 77, (3,), "smallest frame at interval 3"),
    (81, 81, (5,), "smallest frame at interval 5 (odd: the scalar k_gray path, pitch0 = w + 3)"),
    (88, 66, (1,), "near-minimum 4:3 frame, rejected at intervals 3 and 5"),
    (96, 72, (1,), "near-minimum 4:3 frame, rejected at intervals 3 and 5"),
    (321, 241, (5,), "w % 4 == 1"),
    (322, 243, (3,), "w % 4 == 2"),
    (323, 245, (1,), "w % 4 == 3"),
    (279, 211, (5,), "quarter-res width 63 = 2*32 - 1 at scale 0 (partial last cascade tile), qh 46"),
    (280, 216, (5,), "quarter-res width 64 = 2*32 at scale 0 (whole tiles only), qh 48 = 6*8"),
    (285, 220, (5,), "quarter-res width 65 = 2*32 + 1 at scale 0 (a last tile one column wide), qh 49"),
    (1000, 100, (5, 3, 1), "10:1 strip: a single tile row at every scale"),
    (4001, 101, (5, 1), "40:1 strip with an odd width"),
    (16000, 200, (5, 1), "80:1 strip: 500 tiles per row at scale 0, a wide k_gray grid"),
    (100, 1000, (5, 1), "1:10 tall frame: one tile column, many tile rows"),
    (1920, 1080, (5,), "1080p"),
    (2560, 1440, (5,), "1440p"),
    (2579, 1450, (5,), "largest accepted 16:9 frame at interval 5 (2580x1451 is rejected)"),
    (3249, 1827, (1,), "largest 16:9 frame at interval 1 before the first rejected one (3250x1828)"),
    (3864, 2173, (1,), "largest accepted 16:9 frame at interval 1: its largest job, 2732x1536 px, lies in the window "
                       "above 2^22 px where the 32-bit multiplier fits again"),
]

# frames the planner must reject, with the reason it gives
REJECTED = [
    (63, 64, 1, "small"), (64, 63, 2, "small"), (76, 77, 3, "small"), (77, 76, 3, "small"),
    (80, 81, 5, "small"), (81, 80, 5, "small"), (88, 66, 3, "small"), (96, 72, 5, "small"),
    (2580, 1451, 5, "bilinear"), (2733, 1537, 3, "bilinear"), (2896, 1629, 2, "bilinear"), (3250, 1828, 1, "bilinear"),
    (3840, 2160, 5, "bilinear"), (3840, 2160, 3, "bilinear"), (3840, 2160, 2, "bilinear"), (3840, 2160, 1, "bilinear"),
    (36787, 101, 5, "dim"), (101, 36787, 5, "dim"),
]

# the largest entries of GEOMETRIES: one interval and three frames each (the emulation loops over every pixel)
LARGE = {(2560, 1440), (2579, 1450), (3249, 1827), (3864, 2173)}


def geometry_frame(i, W, H, kind="faces"):
    """Frame i of a W x H geometry.  The faces synthesiser cannot place a face in a frame narrower than its smallest
    face, so a tall frame is a column of square face frames."""
    if kind == "faces" and H > 2 * W:
        tiles = [synth.frame(100 * i + k, W, W) for k in range(-(-H // W))]
        return np.ascontiguousarray(np.concatenate(tiles)[:H])
    return synth.frame(i, W, H, kind=kind)


def plan(st, W, H, interval):
    """-> (n_planes, arena_stride, [(off, pitch, w, h, slot, q)]) of build_plan, or None when it rejects the frame"""
    info = np.zeros(2 + 6 * 512, np.int32)
    if st.ht_selftest_planes(W, H, interval, info.ctypes.data, info.size) != 0:
        return None
    n = int(info[0])
    return n, int(info[1]), [tuple(int(v) for v in info[2 + 6 * i: 8 + 6 * i]) for i in range(n)]


# ---------------------------------------------------------------------------------------------------------------------
# accept / reject at the small end

SMALL = sorted(set(range(60, 141, 4)) | {63, 64, 65, 76, 77, 78, 80, 81, 82})


@pytest.mark.parametrize("interval", INTERVALS)
def test_small_frames_are_accepted_exactly_when_the_oracle_accepts_them(st, blob, interval):
    n_acc = n_rej = 0
    for W in SMALL:
        for H in SMALL:
            p = plan(st, W, H, interval)
            f = synth.frame(W * 1000 + H, W, H, kind="noise")
            try:
                oracle.detect(f, blob, interval, 0)
                ok = True
            except RuntimeError:
                ok = False
            assert (p is not None) == ok, (W, H, interval)
            if p is None:
                n_rej += 1
                continue
            n_acc += 1
            pyr = oracle.Pyramid(oracle.grayscale(f), interval)
            g = pyr.geom                                    # (points into pyr: keep pyr alive)
            got = {(slot, q): (w, h) for off, pitch, w, h, slot, q in p[2]}
            assert len(got) == g.n_slots + 3 * (g.n_slots - 2 * g.next), (W, H, interval)
            for s in range(g.n_slots):
                assert got[(s, 0)] == (g.w[s], g.h[s]), (W, H, interval, s)
    assert n_acc and n_rej                                  # the grid straddles the minimum at every interval


# ---------------------------------------------------------------------------------------------------------------------
# the large boundary, restated from the arithmetic

def division_fits(dw, dh):
    """k_resample divides a bilinear numerator n by d = 4 dw dh as (n * M) >> k with n and M in 32 bits.

    The largest numerator is 255 d (four weights summing to d, times 255) plus the rounding half d / 2 = 1022 dw dh,
    and it must fit a uint32.  With M = floor(2^k / d) + 1 the error of n * M / 2^k is n (M d - 2^k) / (d 2^k) <
    n / 2^k, so the quotient is exact for every n <= N once 2^k > (N + 1) d; the planner takes the first such k, and
    then M itself (between N and 2N) must fit 32 bits.  The multiplier, not the numerator, is what binds first:
    dw dh <= 2,968,721 (N = 3.03e9), then again in 4,194,305 .. 4,198,406 where 2^k / d is just below 2^32."""
    d = 4 * dw * dh
    n_max = 255 * d + d // 2
    if n_max >= 1 << 32:
        return False
    k = ((n_max + 1) * d).bit_length()
    return (1 << k) // d + 1 < 1 << 32


def resample_jobs(g):
    """(sx, sy, sw, sh, dw, dh) of every drawImage of src/ccv.js:117-145, the w-2 / h-2 quarter-res copies included"""
    w, h, nxt = list(g.w[:g.n_slots]), list(g.h[:g.n_slots]), g.next
    for s in range(1, g.n_slots):
        src = 0 if s <= g.interval else s - nxt
        yield 0, 0, w[src], h[src], w[s], h[s]                                   # :117-130
        if s >= 2 * nxt:
            yield 1, 0, w[src] - 1, h[src], w[s] - 2, h[s]                       # :135
            yield 0, 1, w[src], h[src] - 1, w[s], h[s] - 2                       # :140
            yield 1, 1, w[src] - 1, h[src] - 1, w[s] - 2, h[s] - 2               # :145


def arena_words(g):
    """Words of one frame quad's arena: every plane 256 B aligned, rows padded to 4 pixels (before the stride's own
    alignment to 64 words)"""
    words = 0
    for s in range(g.n_slots):
        for _ in range(4 if s >= 2 * g.next else 1):
            words = -(-words // 64) * 64 + -(-g.w[s] // 4) * 4 * g.h[s]
    return words


def expected_verdict(W, H, interval):
    """None when the planner must accept W x H, else the limit it exceeds"""
    try:
        g = oracle.geometry(W, H, interval)
    except ValueError:
        return "small"                                      # a 0-sized pyramid level: the reference throws too
    if arena_words(g) > 0x3C000000:
        return "arena"
    for sx, sy, sw, sh, dw, dh in resample_jobs(g):
        if dw <= 0 or dh <= 0 or sw <= 0 or sh <= 0:
            continue                                        # paints nothing
        if dw > 32767 or dh > 32767 or sx + sw > 65535 or sy + sh > 65535:
            return "dim"                                    # tap fractions and source indices are 16-bit
        if not division_fits(dw, dh):
            return "bilinear"
    return None


def test_division_constants_boundary(st):
    """bilinear_division_constants itself (through ht_selftest_ingest, which builds a 1 x q canvas's constants),
    at and around every change of division_fits; the constants the rule admits divide exactly at the worst numerators."""
    st.ht_selftest_ingest.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int]
    edges = [2968721, 4194304, 4198406, 4202512]
    for q in [q + o for q in edges for o in range(-3, 4)]:
        want = division_fits(1, q)
        assert (st.ht_selftest_ingest(None, 0, 1, 1, None, 1, q) == 0) == want, q
        if want:
            d = 4 * q
            n_max = 1022 * q
            k = ((n_max + 1) * d).bit_length()
            M = (1 << k) // d + 1
            for n in (n_max, n_max - 1, n_max - n_max % d - 1, d - 1, d, 2 * d - 1):
                assert (n * M) >> k == n // d, (q, n)
    assert [division_fits(1, q) for q in (2968721, 2968722, 4194304, 4194305, 4198406, 4198407)] == \
        [True, False, False, True, True, False]


LINES = {
    "16:9": [(W, W * 9 // 16) for W in range(2400, 3900)],
    "h=200": [(W, 200) for W in range(18600, 18800)],        # the division limit of a wide strip
    "h=1080": [(W, 1080) for W in range(3400, 3500)],
    "h=101": [(W, 101) for W in range(36700, 36900)],        # dw = floor(W / scale) > 32767 comes first
    "w=101": [(101, H) for H in range(36700, 36900)],
    "w=200": [(200, H) for H in range(18600, 18800)],
}


@pytest.mark.parametrize("line", list(LINES))
def test_planner_limit_is_the_arithmetic_limit(st, line):
    seen = set()
    for interval in INTERVALS:
        for W, H in LINES[line]:
            want = expected_verdict(W, H, interval)
            assert (plan(st, W, H, interval) is not None) == (want is None), (W, H, interval, want)
            seen.add(want)
    assert None in seen and len(seen) >= 2, seen           # every line crosses a limit


def test_boundary_table():
    """The sizes DESIGN.md, INTEGRATION.md and the header state, and the geometry tables' claims."""
    for W, H, intervals, _ in GEOMETRIES:
        for iv in intervals:
            assert expected_verdict(W, H, iv) is None, (W, H, iv)
    for W, H, iv, why in REJECTED:
        assert expected_verdict(W, H, iv) == why, (W, H, iv)
    first_rejected = {5: (2580, 1451), 3: (2733, 1537), 2: (2896, 1629), 1: (3250, 1828)}
    for iv, (W, H) in first_rejected.items():
        assert expected_verdict(W - 1, (W - 1) * 9 // 16, iv) is None
        assert all(expected_verdict(w, w * 9 // 16, iv) is None for w in range(1280, W, 37))
        assert expected_verdict(W, H, iv) == "bilinear" and H == W * 9 // 16
    assert expected_verdict(2880, 1620, 1) is None and expected_verdict(1920, 1080, 5) is None


def test_arena_stride_is_the_layout_sum(st):
    """arena_words (which tests/test_gpu_detect_geometry.py sizes its arena reservations with) is the planner's stride"""
    for W, H, intervals, _ in GEOMETRIES:
        for iv in intervals:
            assert -(-arena_words(oracle.geometry(W, H, iv)) // 64) * 64 == plan(st, W, H, iv)[1], (W, H, iv)


# ---------------------------------------------------------------------------------------------------------------------
# k_gray's 16-bit histogram counters

def largest_cta_share(w, h, chunks):
    """The most pixels of one frame a k_gray CTA counts: CTA b of a quad takes the 4-pixel groups [b * per, (b + 1) *
    per) of the plane rows, pad columns included, and counts only the pixels with col < w (gray_item)."""
    gpr = -(-w // 4)
    n_groups = gpr * h
    per = -(-n_groups // chunks)
    beg = np.arange(chunks, dtype=np.int64) * per
    end = np.minimum(n_groups, beg + per)
    cnt = lambda g: (g // gpr) * w + np.minimum(4 * (g % gpr), w)  # noqa: E731  (pixels in groups [0, g))
    return int((cnt(end) - cnt(beg)).max())


def test_chunk_rule_keeps_every_histogram_counter_below_65536():
    """k_gray's HIST CTAs count two frames in one word, 16 bits each, so a CTA must see fewer than 65,536 pixels of a
    frame.  The host makes chunks >= (w*h + 59999) / 60000 (ht_api.cu, run_detect).  With per = k*gpr + r groups a
    CTA counts at most k*w + 4r pixels, less than per*w/gpr + 3, and per*w/gpr <= w*h/chunks + w/gpr <= 60,004:
    no CTA counts more than 60,006 pixels, however wide the pad columns are against w (w = 65: pitch 68)."""
    worst = 0
    for w in list(range(61, 140)) + [301, 1941, 1942, 1943, 2579, 3249, 3864, 16000]:
        for h in (61, 97, 598, 923, 1051, 1450, 2173):
            chunks = (w * h + 59999) // 60000
            s = largest_cta_share(w, h, chunks)
            assert s <= 60006 and s <= w * h, (w, h, s)
            worst = max(worst, s)
    assert worst > 60000                                    # the sweep reaches the rounding the bound allows
    assert largest_cta_share(1941, 1051, 34) == 60006


# The frames of tests/test_gpu_detect_geometry.py's histogram test: one colour but for a face, the colour being in the
# face template's most common bin, so that the tracked model holds that bin and its weight min(model / cur, 1)
# (src/camshift.js:314-327) depends on how many background pixels the frame histogram counts.
HIST_W, HIST_H = 301, 598           # w % 4 == 1 (k_gray's scalar path); (w*h + 59999) / 60000 = 3 chunks
HIST_BG = (140, 109, 82)            # bin 8:6:5 = 2149 (r >> 4, g >> 4, b >> 4)
HIST_BIN = 2149
HIST_FACES = [(95, 20, 110), (40, 30, 130), (20, 10, 90)]   # x, y, side: the tracker stays in the top 200 rows
OFF_MODEL = (0, 255, 0)             # bin 0:15:0 - no face pixel has g > r


def flat_face(x, y, side, W=HIST_W, H=HIST_H, colour=HIST_BG):
    f = np.empty((H, W, 4), np.uint8)
    f[..., :3] = colour
    f[..., 3] = 255
    t = synth.shim_resize(synth.face_template(), side, side).astype(np.int32)
    f[y:y + side, x:x + side, 0] = t
    f[y:y + side, x:x + side, 1] = (t * 200) >> 8
    f[y:y + side, x:x + side, 2] = (t * 150) >> 8
    return f


def largest_cta_bin(f, chunks):
    """The largest count one k_gray CTA adds to one histogram bin of frame f (the partition of largest_cta_share)"""
    H, W = f.shape[:2]
    gpr = -(-W // 4)
    per = -(-(gpr * H) // chunks)
    px = f[..., :3].astype(np.int64)
    bins = ((px[..., 0] >> 4) << 8) | ((px[..., 1] >> 4) << 4) | (px[..., 2] >> 4)        # rgb_bin
    cta = (np.arange(H)[:, None] * gpr + np.arange(W)[None, :] // 4) // per
    return int(np.bincount((cta * 4096 + bins).ravel()).max())


def oracle_track(f, blob, calc_angles, n_calls=3):
    """detect -> the first most confident rectangle -> initTracker -> n_calls track() in the oracle ->
    (detections, model histogram, the last row any mean-shift window read, [(track object, search window)])"""
    dets = oracle.detect(f, blob)
    cand = None
    for r in dets:
        if cand is None or r[4] > cand[4]:
            cand = r
    ot = oracle.CamshiftTracker(calc_angles=calc_angles)
    ot.init_tracker(f, *[int(math.floor(v)) for v in cand[:4]])
    out, rows = [], 0
    for _ in range(n_calls):
        _, sy, _, sh = ot.search_window()                   # a window keeps its size through a call's iterations
        tr = ot.track(f)
        rows = max(rows, max([sy] + list(tr.wy[:tr.n_iter])) + sh)
        out.append((ot.track_obj(), ot.search_window()))
    return dets, np.ctypeslib.as_array(ot.t.model_hist).copy(), rows, out


@pytest.mark.parametrize("calc_angles", [False, True])
def test_histogram_frames_depend_on_the_background_count(blob, calc_angles):
    """A wrapped 16-bit counter loses 65,536 from the background bin of the frame histogram.  On these frames the
    oracle's result changes when exactly that happens: 65,536 background pixels below every window the tracker reads
    are recoloured into a bin the model does not hold, which changes nothing but the background count.  So the GPU test
    on these frames fails if k_gray's counters wrap."""
    for x, y, side in HIST_FACES:
        f = flat_face(x, y, side)
        assert largest_cta_bin(f, 3) > 60000               # one CTA's background count is at the rule's limit
        dets, model, rows, out = oracle_track(f, blob, calc_angles)
        assert model[HIST_BIN] > 0 and model[0x0F0] == 0
        g = f.copy().reshape(-1, 4)
        g[-65536:, :3] = OFF_MODEL
        g = g.reshape(f.shape)
        first_recoloured_row = HIST_H - (-(-65536 // HIST_W))
        dets2, model2, rows2, out2 = oracle_track(g, blob, calc_angles)
        assert rows <= first_recoloured_row and rows2 <= first_recoloured_row   # no window reads a recoloured pixel
        assert dets2 == dets and np.array_equal(model2, model)
        assert oracle.histogram(g)[HIST_BIN] == oracle.histogram(f)[HIST_BIN] - 65536
        assert out2 != out, (x, y, side)


# ---------------------------------------------------------------------------------------------------------------------
# emulation sweep

EMULATED = [(W, H, iv) for W, H, ivs, _ in GEOMETRIES for iv in (ivs[:1] if (W, H) in LARGE else ivs)]


@pytest.mark.parametrize("W,H,interval", EMULATED)
def test_emulated_detector_equals_the_oracle(st, blob, W, H, interval):
    n = 3 if (W, H) in LARGE else 4
    frames = [geometry_frame(i, W, H) for i in range(n - 1)] + [geometry_frame(n - 1, W, H, kind="noise")]
    arena, info = host_arena(st, frames, W, H, interval)
    pyrs = [oracle.Pyramid(oracle.grayscale(f), interval) for f in frames]
    for i in range(int(info[0])):
        off, pitch, w, h, slot, q = (int(v) for v in info[2 + 6 * i: 8 + 6 * i])
        words = arena[off: off + pitch * h].reshape(h, pitch)
        assert not (words[:, w:] != 0).any(), (slot, q, "pad columns")
        for f in range(4):
            lane = ((words[:, :w] >> (8 * f)) & 0xFF).astype(np.uint8)
            if f < n:
                assert np.array_equal(lane, pyrs[f].plane(slot, q)), (slot, q, f)
            else:
                assert not lane.any(), (slot, q, f, "missing frames are 0")
    cap = 16384
    out = np.zeros((4, cap, 4), np.float64)
    counts = np.zeros(4, np.int32)
    assert st.ht_selftest_cascade(blob, len(blob), W, H, interval, arena.ctypes.data, n, 0, 2, out.ctypes.data,
                                  counts.ctypes.data, cap) == 0
    total = 0
    for f in range(n):
        want = want_raw(frames[f], blob, interval)
        assert counts[f] <= cap
        assert [tuple(out[f, i]) for i in range(counts[f])] == want, f
        total += len(want)
    assert total >= 1                                       # parity must not be vacuous
