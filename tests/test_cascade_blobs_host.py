"""CPU: cascades other than the face model, on the table-driven paths of k_cascade.

parse_cascade (ht_api.cu) sorts every HTC1 blob into one of three paths:
  generated      the face model (blob hash): quad-form truth tables, generated stages, integer late stages
  integer table  every alpha and threshold an 8-digit decimal: ordered fp64 groups {0,1} {2,3} {4,5} {6,7}, then
                 late stages on exact integer sums, decided by the ordered fp64 adds when the sum equals the threshold
  fp table       anything else (or HT_NO_LATE): ordered fp64 groups {0,1} {2,3} {4,5} {6,7,8} {9..} to the end

The corpus (synth.cascade_corpus, whose blobs tests/golden/reference_js_cascades.json embeds) holds tie-prone tenths, 17-digit
numbers, 1 to 9 stages, odd feature shapes, the parser's limits and the face model with one threshold moved by 1e-8.
Here: the oracle equals the reference's own JavaScript on it; every blob takes its path and every malformed one is
refused; the host emulation of k_cascade equals the oracle on every blob; a third, numpy implementation with exact
decimal sums equals the oracle too and shows that the late-stage ties are real and decided both ways; and the
integer decision's premise holds at the parser's limits.
"""
import copy
import ctypes as C
import hashlib
import json
import math
import struct
import sys
from decimal import Decimal
from fractions import Fraction
from pathlib import Path

import numpy as np
import pytest

import oracle
from headtrackr_b200 import synth
from test_cascade_host import run, st  # noqa: F401  (st: the host self-test library fixture)

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tools"))
import pack_cascade  # noqa: E402

from make_goldens_cascades import decode_cascade, rects_digest  # noqa: E402

GOLDEN = json.loads((ROOT / "tests" / "golden" / "reference_js_cascades.json").read_text())
BLOBS = {c["name"]: decode_cascade(c, synth.load_cascade_blob()) for c in GOLDEN["cascades"]}
CASCADES = {name: synth.cascade_from_blob(b) for name, b in BLOBS.items()}   # the src/cascade.js form
HT_ERR_CASCADE = -4
CAP = 16384                                                  # list capacity no frame here reaches
FP_NAMES = {"fp", "limits_alpha", "limits_thr"} | {n for n in CASCADES if n.endswith("_fp")}


@pytest.fixture(scope="module")
def parse(st):
    st.ht_selftest_parse_cascade.argtypes = [C.c_char_p, C.c_size_t, C.c_void_p, C.c_int]

    def f(blob):
        out = np.zeros(16, np.int32)
        rc = st.ht_selftest_parse_cascade(blob, len(blob), out.ctypes.data, out.size)
        if rc != 0:
            return rc, None
        n_groups = int(out[2])
        return 0, dict(fast=int(out[0]), late_int=int(out[1]), n_groups=n_groups, late_first=int(out[3]),
                       group_first=[int(v) for v in out[5: 6 + n_groups]])
    return f


def frames_for(blob, W, H):
    return [synth.frame(i, W, H, blob=blob) for i in range(3)] + [synth.frame(9, W, H, kind="noise")]


def test_corpus_is_the_golden_one():
    """The golden's frames are the ones synth.frame draws from each embedded cascade (the GPU tests generate the same
    corpus with synth.cascade_corpus)."""
    assert set(CASCADES) == set(synth.cascade_corpus())
    for name in CASCADES:
        kind, seed, kw = synth.cascade_corpus()[name]
        assert pack_cascade.pack(synth.cascade(kind, seed, **kw)) == BLOBS[name], name
        assert pack_cascade.pack(CASCADES[name]) == BLOBS[name], name   # the blob read back is the same cascade
        for r in next(x for x in GOLDEN["cascades"] if x["name"] == name)["runs"]:
            frame = synth.frame(r["index"], r["W"], r["H"], blob=BLOBS[name])
            assert hashlib.sha256(np.ascontiguousarray(frame).tobytes()).hexdigest() == r["frame_sha256"], name


@pytest.mark.parametrize("name", sorted(CASCADES))
def test_oracle_equals_reference_js(name):
    runs = next(x for x in GOLDEN["cascades"] if x["name"] == name)["runs"]
    for r in runs:
        frame = synth.frame(r["index"], r["W"], r["H"], blob=BLOBS[name])
        raw = oracle.detect(frame, BLOBS[name], r["interval"], 0, cap=CAP)
        assert (len(raw), rects_digest(raw)) == (r["lists"]["0"]["n"], r["lists"]["0"]["sha256"]), (name, r["W"])
        assert [list(t) for t in oracle.detect(frame, BLOBS[name], r["interval"], 1)] == r["lists"]["1"], (name, r["W"])
        assert raw and r["lists"]["1"], (name, r["W"], r["interval"])    # parity must not be vacuous


def expected_path(name, n_stages, no_late=False):
    if name in FP_NAMES or no_late:
        return dict(fast=0, late_int=0, late_first=n_stages,
                    group_first=[c for c in (0, 2, 4, 6, 9) if c < n_stages] + [n_stages])
    return dict(fast=0, late_int=1, late_first=min(8, n_stages),
                group_first=[c for c in (0, 2, 4, 6) if c < n_stages] + [min(8, n_stages)])


@pytest.mark.parametrize("no_late", [False, True])
def test_every_blob_takes_its_path(parse, no_late, monkeypatch):
    if no_late:
        monkeypatch.setenv("HT_NO_LATE", "1")
    rc, face = parse(synth.load_cascade_blob())
    assert rc == 0
    if no_late:
        assert face == dict(fast=0, late_int=0, n_groups=5, late_first=16, group_first=[0, 2, 4, 6, 9, 16])
    else:
        assert face == dict(fast=1, late_int=1, n_groups=5, late_first=8, group_first=[0, 2, 3, 4, 6, 8])
    for name, blob in BLOBS.items():
        rc, got = parse(blob)
        assert rc == 0, name
        want = expected_path(name, CASCADES[name]["count"], no_late)
        assert got == dict(want, n_groups=len(want["group_first"]) - 1), name
    # the face model rebuilt from its own blob is the face model; one threshold 1e-8 away is not
    assert pack_cascade.pack(synth.cascade_from_blob(synth.load_cascade_blob())) == synth.load_cascade_blob()
    assert parse(BLOBS["near_face"])[1]["fast"] == 0


@pytest.mark.parametrize("sign", [1, -1])
def test_threshold_and_alpha_limits(parse, sign):
    """|threshold| x 1e8 < 2^40 and |alpha| x 1e8 < 2^31 are the integer path's limits, in both signs."""
    for thr, late_int in (("10995.11627775", 1), ("10995.11627776", 0)):
        c = copy.deepcopy(CASCADES["short9"])
        c["stage_classifier"][8]["threshold"] = sign * float(thr)
        assert parse(pack_cascade.pack(c))[1]["late_int"] == late_int, thr
    for a, late_int in (("21.47483647", 1), ("21.47483648", 0)):
        c = copy.deepcopy(CASCADES["short9"])
        c["stage_classifier"][8]["alpha"][0:2] = [-sign * float(a), sign * float(a)]
        assert parse(pack_cascade.pack(c))[1]["late_int"] == late_int, a


def _set(blob, off, fmt, *v):
    b = bytearray(blob)
    struct.pack_into(fmt, b, off, *v)
    return bytes(b)


def test_malformed_blobs_are_refused(parse):
    base = BLOBS["short3"]
    n_st, n_f = struct.unpack_from("<II", base, 4)
    fo = 24 + 16 * n_st
    ao = fo + 32 * n_f
    bad = {
        "magic": b"HTC2" + base[4:],
        "width 20": _set(base, 12, "<I", 20),
        "stage first": _set(base, 24 + 16 + 4, "<I", 0),
        "stage past the features": _set(base, 24 + 16 * (n_st - 1), "<I", 99),
        "stage counts past n_features": _set(base, 8, "<I", n_f - 1),
        "stage counts short of n_features": _set(base, 24, "<I", struct.unpack_from("<I", base, 24)[0] - 1),
        "size 0": _set(base, fo, "<B", 0),
        "size 6": _set(base, fo, "<B", 6),
        "p slot 0 unused": _set(base, fo + 2, "<b", -1),
        "n slot 0 unused": _set(base, fo + 17, "<b", -1),
        "x 24 at level 0": _set(_set(base, fo + 2, "<b", 0), fo + 7, "<B", 24),
        "y 12 at level 1": _set(_set(base, fo + 17, "<b", 1), fo + 27, "<B", 12),
        "x 6 at level 2": _set(_set(base, fo + 2, "<b", 2), fo + 7, "<B", 6),
        "level 3": _set(base, fo + 2, "<b", 3),
        "alpha pair": _set(base, ao, "<dd", -0.5, 0.25),
        "NaN alpha": _set(base, ao, "<dd", math.nan, math.nan),
        "truncated": base[:-1],
        "empty": b"",
    }
    c = copy.deepcopy(CASCADES["short3"])
    c["stage_classifier"] = (c["stage_classifier"] * 22)[:65]
    c["count"] = 65
    bad["65 stages"] = pack_cascade.pack(c)
    c = copy.deepcopy(CASCADES["limits"])
    st0 = c["stage_classifier"][0]
    st0["feature"].append(st0["feature"][0])
    st0["alpha"] += st0["alpha"][:2]
    st0["count"] += 1
    bad["2113 features"] = pack_cascade.pack(c)
    for what, blob in bad.items():
        assert parse(blob)[0] == HT_ERR_CASCADE, what
    # the limits themselves are accepted
    assert parse(BLOBS["limits"])[0] == 0
    assert struct.unpack_from("<II", BLOBS["limits"], 4) == (64, 2112)


@pytest.mark.parametrize("W,H,interval", [(160, 120, 5), (320, 240, 5), (171, 133, 3)])
def test_emulation_equals_the_oracle_on_every_blob(st, W, H, interval):
    for name, blob in BLOBS.items():
        if name.startswith("limits") and W > 200:
            continue                                         # 2112 features: one small frame per blob is enough
        frames = frames_for(blob, W, H)
        want = [[(r[0], r[1], r[2], r[4]) for r in oracle.detect(f, blob, interval, 0, cap=CAP)] for f in frames]
        assert run(st, blob, frames, W, H, interval, cap=CAP) == want, name
        if name not in FP_NAMES:                             # every late decision a tie
            assert run(st, blob, frames, W, H, interval, force_ties=2, cap=CAP) == want, name
        assert all(want[:3]), name


def test_emulation_of_the_face_model_on_the_table_path(st, blob, monkeypatch):
    W, H = 320, 240
    frames = frames_for(blob, W, H)
    want = [[(r[0], r[1], r[2], r[4]) for r in oracle.detect(f, blob, 5, 0)] for f in frames]
    for env in ("HT_NO_FAST", "HT_NO_LATE"):
        monkeypatch.setenv(env, "1")
        assert run(st, blob, frames, W, H) == want, env
        monkeypatch.delenv(env)


# ---- a third implementation: numpy over the oracle's pyramid planes, exact decimal sums beside the fp64 ones ----
def _units(v):
    """v as an integer number of 1e-8, when its shortest decimal literal has at most 8 decimals (else None)."""
    d = Decimal(repr(float(v))) * 100000000
    return int(d) if d == d.to_integral_value() and abs(d) < 2 ** 40 else None


def numpy_cascade(frame, c, interval):
    """src/ccv.js:178-243 vectorised over the windows of a scale and phase.  -> (raw list (x, y, width, conf),
    late-stage ties passed, ties failed).  Decisions are the reference's ordered fp64 sums; where every number of the
    cascade is an 8-digit decimal, the exact integer sum must give the same decision unless it equals the
    threshold (a tie), and the ties of the late stages (>= 8) are counted by their fp64 verdict."""
    pyr = oracle.Pyramid(oracle.grayscale(frame), interval)
    g = pyr.geom
    stages = c["stage_classifier"]
    ints = all(_units(a) is not None for s in stages for a in s["alpha"]) and \
        all(_units(s["threshold"]) is not None for s in stages)
    scale = math.pow(2.0, 1.0 / (interval + 1.0))
    scale_x = 1.0
    out, tie_pass, tie_fail = [], 0, 0
    for i in range(g.scale_upto):
        s0, s1, s2 = i, i + g.next, i + 2 * g.next
        qw, qh = g.w[s2] - 6, g.h[s2] - 6
        for q in range(4 if qw > 0 and qh > 0 else 0):
            dx, dy = q & 1, q >> 1
            planes = (pyr.plane(s0, 0).astype(np.int16), pyr.plane(s1, 0).astype(np.int16), pyr.plane(s2, q).astype(np.int16))

            def px(z, x, y):
                m = 1 << (2 - z)                              # 4, 2, 1 pixels per window step
                o = (2 >> z) if z < 2 else 0
                a = planes[z][dy * o + y: dy * o + y + m * qh: m, dx * o + x: dx * o + x + m * qw: m]
                assert a.shape == (qh, qw)
                return a
            alive = np.ones((qh, qw), bool)
            s = np.zeros((qh, qw))
            for j, stg in enumerate(stages):
                s = np.zeros((qh, qw))
                ex = np.zeros((qh, qw), np.int64)
                for k, f in enumerate(stg["feature"]):
                    pm = np.min([px(z, x, y) for z, x, y in zip(f["pz"], f["px"], f["py"]) if z >= 0], axis=0)
                    nm = np.max([px(z, x, y) for z, x, y in zip(f["nz"], f["nx"], f["ny"]) if z >= 0], axis=0)
                    fire = pm > nm
                    a_fail, a_pass = stg["alpha"][2 * k], stg["alpha"][2 * k + 1]
                    s = s + np.where(fire, a_pass, a_fail)     # one fp64 add per feature, in feature order
                    if ints:
                        ex += np.where(fire, _units(a_pass), _units(a_fail))
                passed = ~(s < stg["threshold"])
                if ints:
                    t = _units(stg["threshold"])
                    tie = ex == t
                    assert np.array_equal((ex > t)[alive & ~tie], passed[alive & ~tie]), (i, q, j)
                    if j >= 8:
                        tie_pass += int((tie & alive & passed).sum())
                        tie_fail += int((tie & alive & ~passed).sum())
                alive &= passed
            for y, x in zip(*np.nonzero(alive)):
                out.append(((x * 4 + dx * 2) * scale_x, (y * 4 + dy * 2) * scale_x, 24 * scale_x, s[y, x]))
        scale_x *= scale
    return out, tie_pass, tie_fail


def test_numpy_cascade_equals_the_oracle_and_ties_go_both_ways(capsys):
    ties = {}
    for name, c in CASCADES.items():
        runs = next(x for x in GOLDEN["cascades"] if x["name"] == name)["runs"]
        for r in runs:
            frame = synth.frame(r["index"], r["W"], r["H"], blob=BLOBS[name])
            got, tp, tf = numpy_cascade(frame, c, r["interval"])
            want = [(t[0], t[1], t[2], t[4]) for t in oracle.detect(frame, BLOBS[name], r["interval"], 0, cap=CAP)]
            assert got == want, (name, r["W"], r["interval"])
            assert got, (name, r["W"], r["interval"])
            t = ties.setdefault(name, [0, 0])
            t[0] += tp
            t[1] += tf
    with capsys.disabled():
        print(f"\nlate-stage exact ties (passed by the fp64 sum, failed by it): {ties}")
    assert ties["ties"][0] >= 30 and ties["ties"][1] >= 30, ties["ties"]


def test_integer_decision_premise_at_the_parser_limits():
    """The late stages decide `exact sum > threshold` on integers (units of 1e-8) where the reference decides
    `!(fp64 sum < fp64 threshold)`.  Both agree whenever the exact sums differ from the threshold if
        |fp64 stage sum - exact decimal sum| + |fp64 threshold - exact threshold| < 1e-8,
    the spacing of the integers.  Bound at the parser's limits (n <= MAX_FEATS features in one stage, |alpha| <= A =
    (2^31 - 1) x 1e-8, |threshold| < 2^40 x 1e-8), with u = 2^-53:
      * each alpha literal is rounded once: |fl(a) - a| <= u |a|, so n u A over the stage;
      * the k-th of the n - 1 adds rounds once: |error| <= u |s_k|, with |s_k| <= k A (1 + u)^n (the partial sum of
        k rounded alphas, grown by at most (1 + u) per add), so u A (1 + u)^n (n (n + 1) / 2 - 1) in all: the worst
        case is every feature in one stage with the same sign;
      * the threshold literal is rounded once: u |T|.
    At n = 2112 that is about 5.3e-9 + 5e-12 + 1.2e-12: below 1e-8 by less than 2x, so raising MAX_FEATS or the alpha
    limit needs a new argument."""
    src = (ROOT / "headtrackr_b200" / "csrc" / "ht_common.cuh").read_text()
    n = int(src.split("constexpr int MAX_FEATS = ")[1].split(";")[0])
    api = (ROOT / "headtrackr_b200" / "csrc" / "ht_api.cu").read_text()
    assert "std::llabs(a_int[k]) > 0x7fffffffll" in api and "std::llabs(r) < (1ll << 40)" in api
    u = Fraction(1, 2 ** 53)
    A = Fraction(2 ** 31 - 1, 10 ** 8)
    T = Fraction(2 ** 40 - 1, 10 ** 8)
    alphas = n * u * A
    adds = u * A * (1 + u) ** n * (Fraction(n * (n + 1), 2) - 1)
    thr = u * T
    total = alphas + adds + thr
    assert total < Fraction(1, 10 ** 8), float(total)
    assert 5.2e-9 < float(adds) < 5.4e-9 and float(total) < 0.54e-8
    # one feature more, or alphas twice as large, and the argument no longer holds
    assert u * 2 * A * (Fraction(n * (n + 1), 2) - 1) > Fraction(1, 10 ** 8)
