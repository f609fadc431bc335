"""CPU: the truncation margin of k_track, against exact-arithmetic moments.

k_track sums the mean-shift moments in a parallel order with FMAs.  Every value the reference truncates - the shift
`(xc - sw/2) >> 0` (src/camshift.js:295-296) and the shape `sqrt(.) << 2` (:237-238) - and the sign of b that picks
the angle's branch (:244) is re-derived from the reference's serial order (moments_serial) when the parallel value
lies within trunc_tolerance (ht_track.cuh) of the decision boundary.  That tolerance must cover the distance between
the two orders' results.  Here:

* exact_moments() sums the window's moments exactly (integer per-bin sums, combined with Fraction), and the derived
  shift / shape / b values follow in exact arithmetic (Decimal for the square roots);
* the oracle's own sums (TrackTrace) are checked against it within the recursive-summation bound gamma_n * m, over the
  synthetic corpus and over the trap frames below;
* trap frames are built so that the exact value of l1 (or of the first shift) sits at k +- delta with delta > 1e-7,
  and the reference's serial sums truncate it on the other side of k - at canvas sizes from 1920x1080 to 3840x2160,
  where the serial error is largest.  Controls of the same construction at 640x480 and 1280x720 pin that error;
* the tolerance k_track would use (ht_selftest_track_tolerance: trunc_tolerance compiled for the host) must exceed twice
  |serial - exact| on every trap, control and corpus pass, and the frame-wide caps it screens with (trunc_cap) must
  exceed the tolerance.

tests/test_gpu_track_margin.py runs the same frames through the kernel.
"""
import ctypes as C
import math
from decimal import Decimal, localcontext
from fractions import Fraction

import numpy as np
import pytest

import oracle
from headtrackr_b200 import synth
from test_cascade_host import st  # noqa: F401  (fixture: the host-only build of ht_api.cu)

U = 2.0 ** -53
MOMENTS = ("m00", "m10", "m01", "m11", "m20", "m02")


def gamma(n):
    return n * U / (1.0 - n * U)


def bins_of(rgba):
    """12-bit colour bin of every pixel (src/camshift.js:49-72)."""
    r, g, b = (rgba[..., i].astype(np.int64) >> 4 for i in range(3))
    return 256 * r + 16 * g + b


# ------------------------------------------------------------------------------------------------------------------
# exact reference

def exact_moments(weights, rgba, window):
    """Exact moments of the window [x0, x1) x [y0, y1) (offsets from its origin), as Fractions.

    Each weight is an fp64 value, so a dyadic rational.  The pixels with a non-zero weight are grouped by colour
    bin; per bin, the integer sums of 1, vx, vy, vx^2, vy^2 and vx*vy are exact in int64 (< 2^63 up to 3840x2160);
    the <= 4096 bins are then combined with Fraction."""
    x0, y0, x1, y1 = window
    if x1 <= x0 or y1 <= y0:
        return {k: Fraction(0) for k in MOMENTS}
    b = bins_of(rgba[y0:y1, x0:x1])
    ys, xs = np.nonzero(weights[b] != 0)
    bb = b[ys, xs]
    order = np.argsort(bb, kind="stable")
    bb, xs, ys = bb[order], xs[order].astype(np.int64), ys[order].astype(np.int64)
    if bb.size == 0:
        return {k: Fraction(0) for k in MOMENTS}
    uniq, start = np.unique(bb, return_index=True)
    sums = {k: np.add.reduceat(v, start) for k, v in
            (("m00", np.ones_like(xs)), ("m10", xs), ("m01", ys), ("m11", xs * ys), ("m20", xs * xs), ("m02", ys * ys))}
    out = {k: Fraction(0) for k in MOMENTS}
    for i, bin_ in enumerate(uniq):
        w = Fraction(float(weights[bin_]))
        for k in MOMENTS:
            out[k] += w * int(sums[k][i])
    return out


def _sqrt(q, prec=60):
    with localcontext() as ctx:
        ctx.prec = prec
        return (Decimal(q.numerator) / Decimal(q.denominator)).sqrt() if q > 0 else Decimal(0)


def exact_values(m, sw, sh, calc_angles):
    """The values the tracker truncates (vxf, vyf, l1, l2) and b, in exact arithmetic (Decimal, 60 digits)."""
    with localcontext() as ctx:
        ctx.prec = 60
        xc, yc = m["m10"] / m["m00"], m["m01"] / m["m00"]
        a = (m["m20"] - m["m10"] * xc) / m["m00"]
        c = (m["m02"] - m["m01"] * yc) / m["m00"]
        b = (m["m11"] - m["m01"] * xc) / m["m00"]
        dec = lambda q: Decimal(q.numerator) / Decimal(q.denominator)  # noqa: E731
        if calc_angles:
            e = _sqrt(4 * b * b + (a - c) * (a - c))
            d = dec(a + c)
            l1 = ((d - e) / 2).sqrt() if d > e else Decimal(0)
            l2 = ((d + e) / 2).sqrt()
        else:
            l1, l2 = _sqrt(a), _sqrt(c)
        return dict(vxf=dec(xc - Fraction(sw, 2)), vyf=dec(yc - Fraction(sh, 2)), l1=l1, l2=l2, b=dec(b))


def serial_values(m, sw, sh, calc_angles):
    """The same values from fp64 moments, with the reference's operations (src/camshift.js:109-120, 230-245)."""
    inv = 1 / m["m00"]
    xc, yc = m["m10"] * inv, m["m01"] * inv
    a = (m["m20"] - m["m10"] * xc) * inv
    c = (m["m02"] - m["m01"] * yc) * inv
    b = (m["m11"] - m["m01"] * xc) * inv
    sq = lambda v: math.sqrt(v) if v >= 0 else math.nan  # noqa: E731
    if calc_angles:
        e = math.sqrt(4 * b * b + (a - c) * (a - c))
        l1, l2 = sq((a + c - e) * 0.5), sq((a + c + e) * 0.5)
    else:
        l1, l2 = sq(a), sq(c)
    return dict(vxf=xc - sw / 2.0, vyf=yc - sh / 2.0, l1=l1, l2=l2, b=b)


def serial_moments(weights, rgba, window):
    """The reference's sums (x outer, y inner, one accumulator, separate multiply and add) - np.cumsum accumulates
    sequentially; pixels of weight 0 add an exact +0.0 and are left out."""
    x0, y0, x1, y1 = window
    pdf = weights[bins_of(rgba[y0:y1, x0:x1])].T          # [x][y]: column-major, as getBackProjectionData
    xs, ys = np.nonzero(pdf)
    val = pdf[xs, ys]
    vx, vy = xs.astype(np.float64), ys.astype(np.float64)
    terms = dict(m00=val, m01=vy * val, m10=vx * val, m11=vx * vy * val, m02=vy * vy * val, m20=vx * vx * val)
    return {k: float(np.cumsum(t)[-1]) if t.size else 0.0 for k, t in terms.items()}


def trunc(v):
    """ES ToInt32 for the magnitudes at hand (NaN -> 0)."""
    return 0 if v != v else int(v)


def dist_int(v):
    return abs(v - round(v))


# ------------------------------------------------------------------------------------------------------------------
# tracking with a trace of every pass

def model_and_weights(A, rect, B):
    ot = oracle.CamshiftTracker(calc_angles=False)
    ot.init_tracker(A, *rect)
    model = np.frombuffer(bytes(ot.t.model_hist), np.uint32)
    return oracle.weights(model, oracle.histogram(B))


def traced_calls(A, rect, B, calc_angles, n_calls):
    """The oracle's track() calls on B after initTracker(A, rect), with the window of every mean-shift pass:
    -> [(trace, [(window, sw, sh, (dx, dy)) per pass], track_obj, search_window)]."""
    H, W = B.shape[:2]
    ot = oracle.CamshiftTracker(calc_angles=calc_angles)
    ot.init_tracker(A, *rect)
    calls = []
    for _ in range(n_calls):
        sx, sy, sw, sh = ot.search_window()
        tr = ot.track(B)
        passes = []
        for i in range(tr.n_iter):
            x0, y0 = max(sx, 0), max(sy, 0)
            win = (x0, y0, min(x0 + sw, W), min(y0 + sh, H))
            nx, ny = tr.wx[i], tr.wy[i]
            passes.append((win, sw, sh, (nx - sx, ny - sy)))
            sx, sy = nx, ny
        calls.append((tr, passes, ot.track_obj(), ot.search_window()))
    return calls


def nonzero_pixels(weights, rgba, window):
    x0, y0, x1, y1 = window
    return int(np.count_nonzero(weights[bins_of(rgba[y0:y1, x0:x1])]))


def tolerance(st, m, n, sw, sh, calc_angles):
    """trunc_tolerance (ht_track.cuh) for fp64 moments m of a window with n non-zero pixels: {vxf, vyf, l1, l2, b}.
    k_track passes an upper bound of n (the area, or m00 / the smallest weight), so its radius is at least this one."""
    mm = (C.c_double * 6)(*[m[k] for k in MOMENTS])
    out = (C.c_double * 5)()
    st.ht_selftest_track_tolerance.argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_double, C.c_int, C.c_void_p]
    st.ht_selftest_track_tolerance(mm, float(n), float(sw), float(sh), int(bool(calc_angles)), out)
    return dict(zip(("vxf", "vyf", "l1", "l2", "b"), out))


# ------------------------------------------------------------------------------------------------------------------
# trap frames

C1, C2 = (0x58, 0xC8, 0x58), (0x58, 0x58, 0xC8)    # the two tracked colours
FILL, BACK = (0x98, 0x98, 0x98), (0xC8, 0x38, 0x38)  # A's other colour (absent from B), B's background (absent from A)


def _rgba(W, H, colour):
    f = np.empty((H, W, 4), np.uint8)
    f[..., :3] = colour
    f[..., 3] = 255
    return f


def trap_frames(W, H, cA, cols):
    """Frame A: cA[0] pixels of C1 then cA[1] of C2 (raster order) on FILL.  Frame B: on BACK, a one-pixel column of
    C1 at cols[0] = (x, y0, h) and one of C2 at cols[1].  Tracked from a rect that covers A, each column's weight is
    cA[i] / h[i]: non-dyadic unless h[i] divides cA[i] * 2^k."""
    A = _rgba(W, H, FILL)
    flat = A.reshape(-1, 4)
    flat[:cA[0], :3] = C1
    flat[cA[0]:cA[0] + cA[1], :3] = C2
    B = _rgba(W, H, BACK)
    for colour, (x, y0, h) in zip((C1, C2), cols):
        B[y0:y0 + h, x, :3] = colour
    return A, B


def _column_sums(cA, cols):
    """Exact moments of the two columns over the canvas (closed forms), and the serial fp64 sums."""
    ex = {k: Fraction(0) for k in MOMENTS}
    terms = {k: [] for k in MOMENTS}
    for c, (x, y0, h) in zip(cA, cols):
        w = c / h
        fw = Fraction(w)
        vx = x
        vy = np.arange(y0, y0 + h, dtype=np.float64)
        s1, s2 = (y0 + y0 + h - 1) * h // 2, sum(j * j for j in range(y0, y0 + h))
        ex["m00"] += fw * h; ex["m10"] += fw * h * vx; ex["m20"] += fw * h * vx * vx
        ex["m01"] += fw * s1; ex["m11"] += fw * s1 * vx; ex["m02"] += fw * s2
        val = np.full(h, w)
        fvx = float(vx)
        terms["m00"].append(val); terms["m10"].append(fvx * val); terms["m20"].append(fvx * fvx * val)
        terms["m01"].append(vy * val); terms["m11"].append(fvx * vy * val); terms["m02"].append(vy * vy * val)
    ser = {k: float(np.cumsum(np.concatenate(v))[-1]) for k, v in terms.items()}
    return ex, ser


# One family per row: canvas, init-rect width (the window stays the canvas while the search window only moves left
# or up), x of the first column, calc_angles, and sym: columns of equal height (exact b == 0).
FAMILIES = {
    "1080p_wide": dict(W=1920, H=1080, rect_w=3840, anchor=1850, calc=False, sym=False),
    "1440p": dict(W=2560, H=1440, rect_w=2560, anchor=1279, calc=False, sym=False),
    "1440p_odd": dict(W=2562, H=1440, rect_w=2562, anchor=1280, calc=False, sym=False),
    "4k": dict(W=3840, H=2160, rect_w=3840, anchor=1919, calc=False, sym=False),
    "4k_angles": dict(W=3840, H=2160, rect_w=3840, anchor=1919, calc=True, sym=False),
    "4k_symmetric": dict(W=3840, H=2160, rect_w=3840, anchor=1919, calc=True, sym=True),
    "4k_wide": dict(W=3840, H=2160, rect_w=7680, anchor=3700, calc=False, sym=False),
}
# controls: the same construction at the sizes the suite tracks at elsewhere
CONTROLS = {
    "480p": dict(W=640, H=480, rect_w=640, anchor=319, calc=False, sym=False),
    "480p_angles": dict(W=640, H=480, rect_w=640, anchor=319, calc=True, sym=False),
    "720p": dict(W=1280, H=720, rect_w=1280, anchor=639, calc=False, sym=False),
    "720p_wide": dict(W=1280, H=720, rect_w=2560, anchor=1200, calc=False, sym=True),
}
MIN_DELTA = 1e-7      # the exact value is further than this from the integer it truncates across
SHIFT_GAP = 1e-4      # every shift of every pass is at least this far from an integer


def _candidates(fam):
    """Deterministic candidate order: column gap, heights, then the two masses around the ratio that puts l1 at 1."""
    W, H = fam["W"], fam["H"]
    for d in (2, 4):
        for dh in ((0, 0),) if fam["sym"] else ((0, 1), (0, 7), (0, 30)):
            h1, h2 = H - dh[0], H - dh[1]
            for total in range(400, 4000, 7):
                if d == 2:
                    pairs = [(total // 2, total - total // 2)]
                else:                       # 4 sqrt(m1 m2) / (m1 + m2) = 1  <=>  m1 / m2 = 7 + sqrt(48)
                    m2 = round(total / (8 + math.sqrt(48)))
                    pairs = [(total - m2 + s, m2 - s) for s in (-1, 0, 1)]
                for m1, m2 in pairs:
                    for cA in ((m1, m2), (m2, m1)):
                        if fam["sym"] and d == 2 and cA[0] == cA[1]:
                            continue
                        yield d, (cA[0], cA[1]), ((fam["anchor"], 0, h1), (fam["anchor"] + d, 0, h2))


def _prefilter(fam, cA, cols, control):
    """Closed-form check that the columns make a trap (a control: a valid frame): -> the truncated name or None."""
    W, H = fam["W"], fam["H"]
    for c, (_, _, h) in zip(cA, cols):
        den = Fraction(c, h).denominator
        if c >= h or den & (den - 1) == 0:     # a weight of 1, or a dyadic one
            return None
    ex, ser = _column_sums(cA, cols)
    e = exact_values(ex, fam["rect_w"], H, fam["calc"])
    s = serial_values(ser, fam["rect_w"], H, fam["calc"])
    for k in ("vxf", "vyf"):
        if float(e[k]) >= 1 or dist_int(float(e[k])) < SHIFT_GAP:
            return None
    if control:
        return "l1"
    for k in ("l1", "l2"):
        if dist_int(e[k]) > MIN_DELTA and trunc(s[k]) != math.floor(e[k]):
            return k
    return None


_TRAPS = {}

# A trap on the shift instead: every pixel of a 3840x2160 canvas has a non-zero weight - columns [0, k) one colour,
# [k, W) the other - so the serial sums run over 8.3 M terms, and the masses put the exact xc - W/2 at s0 +- delta.
# s0 = +1: a shift of 1 or 0 moves the window or not, so the outputs show which way it was truncated.
SHIFT_FAMILIES = {"4k_shift": dict(W=3840, H=2160, k=1000, m2=1500000, s0=1)}


def _egcd(a, b):
    if b == 0:
        return a, 1, 0
    g, x, y = _egcd(b, a % b)
    return g, y, x - (a // b) * y


def _shift_candidates(fam):
    """Masses with cA1 P - cA2 Q = j, where P / 2 and Q / 2 are the two regions' mass centres' distances from
    W/2 + s0: the exact xc - W/2 is then s0 + j / (2 (cA1 + cA2))."""
    W, k, s0 = fam["W"], fam["k"], fam["s0"]
    P, Q = k - 1 - 2 * s0, W + 2 * s0 - k + 1
    g, x, y = _egcd(P, Q)
    assert g == 1
    for j in (2, -2, 3, -3, 4, -4, 5, -5):
        for s in range(8):
            # cA1 = j x + t Q, cA2 = -j y + t P, with cA2 near m2 + s * P
            t = (fam["m2"] + j * y) // P + s
            yield j * x + t * Q, -j * y + t * P


def _find_shift_trap(name):
    fam = SHIFT_FAMILIES[name]
    W, H, k = fam["W"], fam["H"], fam["k"]
    rect = (0, 0, W, H)
    for cA1, cA2 in _shift_candidates(fam):
        A = _rgba(W, H, FILL)
        flat = A.reshape(-1, 4)
        flat[:cA1, :3] = C1
        flat[cA1:cA1 + cA2, :3] = C2
        B = _rgba(W, H, C1)
        B[:, :k, :3] = C2
        w = model_and_weights(A, rect, B)
        win = (0, 0, W, H)
        e = exact_values(exact_moments(w, B, win), W, H, False)
        if not MIN_DELTA < dist_int(e["vxf"]) < 1e-5:
            continue
        (tr, passes, obj, _), = traced_calls(A, rect, B, False, 1)
        if passes[0][3][0] != trunc(float(e["vxf"])):   # the oracle's first shift crosses the integer
            return dict(name=name, A=A, B=B, rect=rect, calc=False, key="vxf", cA=(cA1, cA2), control=False)
    return None


def find_trap(name):
    """The first candidate of a family that is a trap, confirmed through the oracle: -> dict."""
    if name in _TRAPS:
        return _TRAPS[name]
    if name in SHIFT_FAMILIES:
        _TRAPS[name] = _find_shift_trap(name)
        return _TRAPS[name]
    fam = {**FAMILIES, **CONTROLS}[name]
    control = name in CONTROLS
    found = None
    for d, cA, cols in _candidates(fam):
        key = _prefilter(fam, cA, cols, control)
        if key is None:
            continue
        A, B = trap_frames(fam["W"], fam["H"], cA, cols)
        found = dict(name=name, A=A, B=B, rect=(0, 0, fam["rect_w"], fam["H"]), calc=fam["calc"], key=key, cA=cA,
                     cols=cols, control=control)
        if control or _confirm(found):
            break
        found = None
    _TRAPS[name] = found
    return found


def _confirm(t):
    """The oracle's first call truncates the trap value across k, and the first exact pass has no close shift."""
    (tr, passes, obj, win), = traced_calls(t["A"], t["rect"], t["B"], t["calc"], 1)
    w = model_and_weights(t["A"], t["rect"], t["B"])
    win0, sw, sh, _ = passes[-1]
    e = exact_values(exact_moments(w, t["B"], win0), sw, sh, t["calc"])
    got = obj["width"] if t["key"] == "l1" else obj["height"]
    return got != 4 * math.floor(e[t["key"]]) and dist_int(e[t["key"]]) > MIN_DELTA


# ------------------------------------------------------------------------------------------------------------------
# tests

def caps(st, W, H, sw, sh, l1, l2):
    """The frame-wide caps k_track screens each decision with before it computes the window's radius."""
    out = (C.c_double * 5)()
    st.ht_selftest_track_cap.argtypes = [C.c_int, C.c_int] + [C.c_double] * 4 + [C.c_void_p]
    st.ht_selftest_track_cap(W, H, float(sw), float(sh), float(l1), float(l2), out)
    return dict(zip(("vxf", "vyf", "l1", "l2", "b"), out))


def _check_calls(st, A, rect, B, calc, n_calls, margins=None):
    """Every pass of every call: the oracle's sums are within gamma_n * m of exact, every truncation the oracle made
    agrees with the exact value unless that value is within the tolerance of an integer, the tolerance covers twice
    |serial - exact| of every value it guards, and the frame's caps are at least the tolerance of any pixel count."""
    w = model_and_weights(A, rect, B)
    calls = traced_calls(A, rect, B, calc, n_calls)
    for ci, (tr, passes, obj, _) in enumerate(calls):
        for pi, (win, sw, sh, (dx, dy)) in enumerate(passes):
            ex = exact_moments(w, B, win)
            if ex["m00"] == 0:
                continue
            ser = serial_moments(w, B, win)
            area = (win[2] - win[0]) * (win[3] - win[1])
            if pi == len(passes) - 1:   # the oracle's final moments are those of this window
                for k in MOMENTS:
                    assert getattr(tr, k) == ser[k], (ci, k)
                    assert abs(Fraction(getattr(tr, k)) - ex[k]) <= Fraction(gamma(area)) * ex[k], (ci, k)
            e = exact_values(ex, sw, sh, calc)
            s = serial_values(ser, sw, sh, calc)
            tol = tolerance(st, ser, nonzero_pixels(w, B, win), sw, sh, calc)
            keys = ("vxf", "vyf", "l1", "l2", "b") if pi == len(passes) - 1 else ("vxf", "vyf")
            tol_area = tolerance(st, ser, area, sw, sh, calc)
            cap = caps(st, B.shape[1], B.shape[0], sw, sh, s["l1"], s["l2"])
            for k in keys:
                assert tol[k] <= tol_area[k] <= cap[k] or s[k] != s[k], (ci, pi, k, tol_area[k], cap[k])
                err = abs(Decimal(s[k]) - e[k]) if s[k] == s[k] else Decimal(0)
                assert 2 * err <= Decimal(tol[k]), (ci, pi, k, err, tol[k])
                if margins is not None:
                    margins[k] = max(margins.get(k, 0.0), float(err))
            # the oracle's shift is the serial value's truncation; it equals the exact one unless that is within
            # the tolerance of an integer
            if dist_int(e["vxf"]) > tol["vxf"]:
                assert dx == trunc(float(e["vxf"])), (ci, pi)
            if dist_int(e["vyf"]) > tol["vyf"]:
                assert dy == trunc(float(e["vyf"])), (ci, pi)
    return calls


@pytest.mark.parametrize("name", list(FAMILIES))
def test_trap_frame_truncates_across_an_integer(st, name):
    """The family has a trap: the exact shape value is k +- delta (delta > 1e-7), the oracle truncates it on the other
    side of k, every shift is >= 1e-4 from an integer (so only the shape decision can take the fallback), and the
    kernel's tolerance covers the serial error."""
    t = find_trap(name)
    assert t is not None, name
    (tr, passes, obj, _), = traced_calls(t["A"], t["rect"], t["B"], t["calc"], 1)
    w = model_and_weights(t["A"], t["rect"], t["B"])
    H, W = t["B"].shape[:2]
    for win, sw, sh, _ in passes:
        assert win == (0, 0, W, H)                      # the window is the canvas on every pass
        e = exact_values(exact_moments(w, t["B"], win), sw, sh, t["calc"])
        assert dist_int(e["vxf"]) >= SHIFT_GAP and dist_int(e["vyf"]) >= SHIFT_GAP
    ex = exact_moments(w, t["B"], passes[-1][0])
    e = exact_values(ex, passes[-1][1], passes[-1][2], t["calc"])
    k = t["key"]
    assert dist_int(e[k]) > MIN_DELTA
    got = (obj["width"] if k == "l1" else obj["height"]) // 4
    assert got != math.floor(e[k])                     # the reference truncates across k
    if FAMILIES[name]["sym"]:
        assert e["b"] == 0
    ser = {k2: getattr(tr, k2) for k2 in MOMENTS}
    s = serial_values(ser, passes[-1][1], passes[-1][2], t["calc"])
    tol = tolerance(st, ser, nonzero_pixels(w, t["B"], passes[-1][0]), passes[-1][1], passes[-1][2], t["calc"])
    assert 2 * abs(Decimal(s[k]) - e[k]) <= Decimal(tol[k])
    _check_calls(st, t["A"], t["rect"], t["B"], t["calc"], 3)


@pytest.mark.parametrize("name", list(SHIFT_FAMILIES))
def test_shift_trap_frame_truncates_across_an_integer(st, name):
    """8.3 M non-zero pixels: the exact first shift is s0 +- delta (delta > 1e-7), the oracle truncates it on the other
    side, and the tolerance covers twice the serial error of every value of every pass."""
    t = find_trap(name)
    assert t is not None, name
    (tr, passes, obj, _), = traced_calls(t["A"], t["rect"], t["B"], False, 1)
    w = model_and_weights(t["A"], t["rect"], t["B"])
    win, sw, sh, (dx, dy) = passes[0]
    e = exact_values(exact_moments(w, t["B"], win), sw, sh, False)
    assert dist_int(e["vxf"]) > MIN_DELTA and round(e["vxf"]) == SHIFT_FAMILIES[name]["s0"]
    assert dx != trunc(float(e["vxf"]))
    _check_calls(st, t["A"], t["rect"], t["B"], False, 2)


# |serial - exact| of the control frames' values: pinned, so that a change of the construction or of the reference's
# order shows up here.  They are below 1e-7 (the radius the kernel used before the tolerance followed the window).
CONTROL_MAX_ERR = 1e-7


@pytest.mark.parametrize("name", list(CONTROLS))
def test_control_frames_serial_error(st, name):
    t = find_trap(name)
    margins = {}
    _check_calls(st, t["A"], t["rect"], t["B"], t["calc"], 3, margins)
    assert 0 < margins["l1"] < CONTROL_MAX_ERR, margins


def _face_rect(blob, f):
    res = oracle.detect(f, blob)
    best = max(res, key=lambda r: r[4])
    return [int(math.floor(v)) for v in best[:4]]


@pytest.mark.parametrize("W,H,idx,calc", [(320, 240, 0, True), (320, 240, 1, False), (640, 480, 2, True),
                                          (640, 480, 3, False), (1280, 720, 4, True), (1280, 720, 5, False)])
def test_exact_reference_agrees_with_oracle_on_the_corpus(st, blob, W, H, idx, calc):
    """Synthetic faces: on every pass of 5 track() calls the oracle's sums are within gamma_n * m of exact, and the
    tolerance covers twice |serial - exact| of every truncated value."""
    f = synth.frame(idx, W, H)
    _check_calls(st, f, _face_rect(blob, f), f, calc, 5)


def test_tolerance_covers_a_full_canvas_of_nonzero_weights(st):
    """The largest sums the tracker makes: every pixel of a 3840x2160 canvas has a non-zero, non-dyadic weight."""
    W, H = 3840, 2160
    A = _rgba(W, H, C1)
    A.reshape(-1, 4)[:W * H // 3, :3] = C2
    B = _rgba(W, H, C1)
    B[:, :W // 3 + 5, :3] = C2
    rect = (0, 0, W, H)
    w = model_and_weights(A, rect, B)
    win = (0, 0, W, H)
    ex = exact_moments(w, B, win)
    ser = serial_moments(w, B, win)
    for calc in (False, True):
        e, s = exact_values(ex, W, H, calc), serial_values(ser, W, H, calc)
        tol = tolerance(st, ser, W * H, W, H, calc)
        for k in ("vxf", "vyf", "l1", "l2", "b"):
            assert 2 * abs(Decimal(s[k]) - e[k]) <= Decimal(tol[k]), (calc, k)
