"""GPU: k_group and the VJ->CS hand-off on crowded frames (tests/test_group_crowd_host.py's CROWD), against the oracle.

Frames with a few faces leave most of k_group unexercised: one pass of each lane loop, one 32-entry ballot block in
steps 3 and 4, small components, no ties.  The crowds here give 200 to 2,000 raw windows and 70 to 500 groups.

  * detection: raw lists (debug_raw) and grouped lists bit-exact at every interval and min_neighbors 0 to 8, in batches
    that mix crowded, noise and empty frames in the same quads; again under forced ties and without TMA;
  * truncation: a list longer than max_rects_per_frame is the reference's first K entries with HT_WARN_OVERFLOW; a raw
    list longer than max_raw_per_frame is a subsequence of the reference's;
  * hand-off: at the default K = 64 and at K = 1, ht_detect_track, ht_stream_step, ht_tracker_step and ht_tracker_feed
    seed the face src/facetrackr.js picks from the WHOLE grouped list, also when it lies past index K - 1;
    ht_track_init_from_detect picks from the list the caller passes.
Each test makes its own contexts and closes them.
"""
import math

import numpy as np
import pytest

import oracle
from headtrackr_b200 import Context, synth
from test_group_crowd_host import CROWD, crowd, first_max

pytestmark = pytest.mark.gpu

BIG = 16384                  # list capacities that no crowd here reaches


def tup(d):
    return (d["x"], d["y"], d["width"], d["height"], d["confidence"], d.get("neighbors", d.get("neighbor")))


def context(W, H, n, raw=BIG, K=BIG):
    return Context(max_width=W, max_height=H, max_frames=n, max_raw_per_frame=raw, max_rects_per_frame=K)


def raw_lists(c, n):
    out = []
    for f in range(n):
        r, cnt = c.debug_raw(f, cap=BIG)
        assert cnt == len(r), (f, cnt)
        out.append(r)
    return out


def empty(W, H):
    return synth.frame(0, W, H, kind="constant")


# per geometry: the batch (crowds mixed with noise and empty frames inside the same quads) and the intervals
BATCHES = {
    (160, 120): (["small", "noise", "small_b", "empty", "small"], (1, 2, 3, 5)),
    (320, 240): (["beyond_k", "noise", "tied_max", "empty", "two_sizes", "nested", "edges", "chains", "grid_ties"],
                 (1, 2, 3, 5)),
    (640, 480): (["vga", "empty", "noise", "vga_b", "vga"], (2, 5)),
    (1280, 720): (["hd", "noise", "hd"], (3, 5)),
}
MIN_NEIGHBORS = (0, 1, 2, 3, 5, 8)


def batch_frames(W, H):
    names, _ = BATCHES[(W, H)]
    out = []
    for nm in names:
        if nm == "noise":
            out.append(synth.frame(7, W, H, kind="noise"))
        elif nm == "empty":
            out.append(empty(W, H))
        elif nm.endswith("_b"):                              # the same recipe with another seed
            Wc, Hc, kw = CROWD[nm[:-2]]
            out.append(synth.crowd_frame(W=Wc, H=Hc, **dict(kw, seed=kw["seed"] + 10)))
        else:
            assert CROWD[nm][:2] == (W, H)
            out.append(crowd(nm))
    return np.stack(out)


@pytest.mark.parametrize("W,H", list(BATCHES))
def test_crowded_detection_equals_the_oracle(blob, W, H):
    frames = batch_frames(W, H)
    n = len(frames)
    _, intervals = BATCHES[(W, H)]
    c = context(W, H, n)
    try:
        longest = 0
        for iv in intervals:
            raws = [oracle.detect(f, blob, iv, 0, cap=BIG) for f in frames]
            for mn in MIN_NEIGHBORS:
                got = c.detect(frames, iv, mn)
                assert c.last_warning is None, (iv, mn)
                if mn == 0:
                    assert raw_lists(c, n) == raws, iv
                for i in range(n):
                    want = raws[i] if mn == 0 else oracle.group(raws[i], mn, cap=BIG)
                    assert [tup(d) for d in got[i]] == want, (iv, mn, i)
                    longest = max(longest, len(want) if mn else 0)
        assert longest >= (33 if W >= 320 else 16)            # more than one ballot block in k_group's steps 3 and 4
    finally:
        c.close()


@pytest.mark.parametrize("variant", ["ties1", "ties2", "ties3", "no_tma"])
def test_crowded_detection_through_the_fallbacks(blob, variant, monkeypatch):
    """Two crowds under forced exactness fallbacks (dense survivor sets through the tie paths) and without TMA."""
    for name in ("beyond_k", "vga"):
        W, H, _ = CROWD[name]
        f = crowd(name)
        frames = np.stack([f, synth.frame(3, W, H, kind="noise"), f, f, f])
        raw = oracle.detect(f, blob, 5, 0, cap=BIG)
        with monkeypatch.context() as m:
            if variant == "no_tma":
                m.setenv("HT_TMA", "0")
            c = context(W, H, len(frames))
        try:
            if variant.startswith("ties"):
                c.debug_set_exactness(int(variant[-1]))
            for mn in (0, 1, 3):
                got = c.detect(frames, 5, mn)
                assert c.last_warning is None
                want = raw if mn == 0 else oracle.group(raw, mn, cap=BIG)
                for i in (0, 2, 3, 4):
                    assert [tup(d) for d in got[i]] == want, (name, mn, i)
            assert raw_lists(c, len(frames))[4] == raw
        finally:
            c.close()


# ---- truncation contracts ----

@pytest.mark.parametrize("K", [1, 8, 64])
def test_list_longer_than_k_is_the_reference_prefix(blob, K):
    f = crowd("vga")
    W, H, _ = CROWD["vga"]
    raw = oracle.detect(f, blob, 5, 0, cap=BIG)
    frames = np.stack([f, empty(W, H)])
    c = context(W, H, 2, raw=BIG, K=K)
    try:
        for mn in (0, 1, 3):
            want = raw if mn == 0 else oracle.group(raw, mn, cap=BIG)
            assert len(want) > K
            got = c.detect(frames, 5, mn)
            assert c.last_warning is not None and "overflow" in c.last_warning, mn
            assert [tup(d) for d in got[0]] == want[:K] and got[1] == [], mn
        # a frame whose lists fit: no warning
        got = c.detect(np.stack([empty(W, H), empty(W, H)]), 5, 1)
        assert c.last_warning is None and got == [[], []]
    finally:
        c.close()


@pytest.mark.parametrize("raw_cap", [64, 1024])
def test_raw_list_longer_than_its_capacity_is_a_subsequence(blob, raw_cap):
    f = crowd("vga")
    W, H, _ = CROWD["vga"]
    raw = oracle.detect(f, blob, 5, 0, cap=BIG)
    assert len(raw) > raw_cap
    c = context(W, H, 1, raw=raw_cap, K=BIG)
    try:
        c.detect(f[None], 5, 1)
        assert c.last_warning is not None and "overflow" in c.last_warning
        got, cnt = c.debug_raw(0, cap=BIG)
        assert cnt == len(raw) and len(got) == raw_cap
        pos = {r: i for i, r in enumerate(raw)}
        idx = [pos[r] for r in got]                           # every entry is one of the reference's ...
        assert all(a < b for a, b in zip(idx, idx[1:]))       # ... in the reference's order
    finally:
        c.close()
    c = context(W, H, 1, raw=len(raw), K=BIG)                 # exactly enough: no warning
    try:
        c.detect(f[None], 5, 1)
        assert c.last_warning is None and raw_lists(c, 1)[0] == raw
    finally:
        c.close()


# ---- the VJ->CS hand-off ----

HANDOFF = ["beyond_k", "tied_max", "grid_ties"]


def pick(blob, f):
    """facetrackr's VJ result on frame f: the first maximum over the whole grouped list (src/facetrackr.js:157-165)"""
    g = oracle.detect(f, blob, 5, 1, cap=BIG)
    return g[first_max(g)]


def oracle_track(f, rect, calc_angles, n_calls):
    ot = oracle.CamshiftTracker(calc_angles=calc_angles)
    ot.init_tracker(f, *[int(math.floor(v)) for v in rect[:4]])
    for _ in range(n_calls):
        ot.track(f)
    return ot


def assert_obj(obj, ot, what):
    w = ot.track_obj()
    assert (obj["x"], obj["y"], obj["width"], obj["height"]) == (w["x"], w["y"], w["width"], w["height"]), what
    assert abs(obj["angle"] - w["angle"]) <= 1e-4 or (math.isnan(obj["angle"]) and math.isnan(w["angle"])), what


def test_handoff_corpus_needs_the_whole_list(blob):
    """beyond_k's pick lies past index 63; the tied frames' pick is the first of several maxima."""
    g = oracle.detect(crowd("beyond_k"), blob, 5, 1, cap=BIG)
    assert first_max(g) > 63 and first_max(g[:64]) != first_max(g)
    for name in ("tied_max", "grid_ties"):
        g = oracle.detect(crowd(name), blob, 5, 1, cap=BIG)
        assert sum(r[4] == g[first_max(g)][4] for r in g) >= 2


@pytest.mark.parametrize("K", [0, 1])                       # 0: the default, 64
@pytest.mark.parametrize("pipelined", [False, True])
def test_detect_track_seeds_the_reference_face(blob, K, pipelined):
    import torch
    W, H = 320, 240
    frames = np.stack([crowd(n) for n in HANDOFF] + [empty(W, H)])
    n = len(frames)
    c = context(W, H, n, raw=BIG, K=K)
    try:
        assert c.K == (K or 64)
        if not pipelined:
            dets, found, objs, wins = c.detect_track(frames, 5, 1, calc_angles=False, n_calls=3)
            assert c.last_warning is not None                 # the crowds' lists are longer than K
        else:
            c.set_pipeline(True)
            dev = torch.from_numpy(frames).cuda()
            outs = (torch.zeros((n, c.K, 6), dtype=torch.float64, device="cuda"),
                    torch.zeros((n,), dtype=torch.int32, device="cuda"), torch.zeros((n,), dtype=torch.int32, device="cuda"),
                    torch.zeros((n, 6), dtype=torch.int32, device="cuda"), torch.zeros((n, 4), dtype=torch.int32, device="cuda"))
            torch.cuda.synchronize()
            for _ in range(3):                                # call s+1's k_group runs behind call s's tracking
                c.detect_track(dev, 5, 1, calc_angles=False, n_calls=3, outputs=outs)
            c.sync()
            assert c.last_warning is not None
            found = outs[2].cpu().tolist()
            o = outs[3].cpu().numpy()
            objs = [dict(x=int(r[0]), y=int(r[1]), width=int(r[2]), height=int(r[3]),
                         angle=float(r[4:6].copy().view(np.float64)[0])) for r in o]
            wins = [tuple(int(v) for v in r) for r in outs[4].cpu().numpy()]
        for i, name in enumerate(HANDOFF):
            ot = oracle_track(frames[i], pick(blob, frames[i]), False, 3)
            assert found[i] == 1, name
            assert_obj(objs[i], ot, name)
            assert wins[i] == ot.search_window(), name
            _, fo, obj_o = oracle.detect_track(frames[i], blob, 5, 1, n_calls=3)
            assert fo == 1 and obj_o["x"] == objs[i]["x"] and obj_o["y"] == objs[i]["y"], name
        assert found[n - 1] == 0
    finally:
        c.close()


@pytest.mark.parametrize("K", [0, 1])
def test_stream_step_seeds_the_reference_face(blob, K):
    W, H = 320, 240
    frames = np.stack([crowd(n) for n in HANDOFF] + [empty(W, H)])
    c = context(W, H, len(frames), raw=BIG, K=K)
    try:
        c.stream_reset()
        ev = c.stream_step(frames)
        ev2 = c.stream_step(frames)
        for i, name in enumerate(HANDOFF):
            p = pick(blob, frames[i])
            e = ev[i]
            assert e["detection"] == "VJ" and e["found"], name
            assert (e["x"], e["y"], e["width"], e["height"], e["confidence"]) == tuple(p[:5]), name
            ot = oracle_track(frames[i], p, False, 1)
            assert ev2[i]["detection"] == "CS", name
            assert_obj(ev2[i], ot, name)
        assert ev[-1]["detection"] == "VJ" and not ev[-1]["found"] and ev2[-1]["detection"] == "VJ"
    finally:
        c.close()


def host_lifecycle(blob, frames, n_ticks):
    """main.Tracker over the oracle (tests/test_host_lifecycle.py's harness): per frame, per tick, the events"""
    from headtrackr_b200 import Canvas, main
    from test_host_logic import OracleBackend
    out = []
    for f in frames:
        H, W = f.shape[:2]
        video, canvas = Canvas(f), Canvas(np.zeros((H, W, 4), np.uint8))
        clock = [1.0e12]
        ht = main.Tracker(dict(ui=False), backend=OracleBackend(blob), clock=lambda: clock[0])
        log = []
        for t in ("headtrackrStatus", "facetrackingEvent", "headtrackingEvent"):
            ht.addEventListener(t, log.append)
        ht.init(video, canvas, False)
        ticks = []
        for t in range(n_ticks):
            clock[0] += 35.0
            n0 = len(log)
            if t == 0:
                assert ht.start() is True
            else:
                ht.step()
            ticks.append([{k: v for k, v in e.items() if k != "time"} for e in log[n0:]])
        out.append(ticks)
    return out


@pytest.mark.parametrize("K", [0, 1])
@pytest.mark.parametrize("entry", ["step", "feed"])
def test_tracker_seeds_the_reference_face(blob, K, entry):
    """The whitebalance gate (15 equal frames), VJ on the crowd, then CS: every event equals the host lifecycle over the
    oracle, tick by tick."""
    from headtrackr_b200.streams import TrackerSet
    from test_host_main import check_events
    W, H = 320, 240
    frames = [crowd(n) for n in HANDOFF]
    T = 19
    want = host_lifecycle(blob, frames, T)
    c = context(W, H, len(frames), raw=BIG, K=K)
    try:
        ts = TrackerSet(c, len(frames), {})
        log = [[] for _ in frames]
        ts.addEventListener(lambda k, e: log[k].append(e))
        vj_seen = 0
        for t in range(T):
            marks = [len(l) for l in log]
            if t == 0:
                ts.start()
            if entry == "step":
                recs = ts.step(np.stack(frames), now_ms=1.0e12 + 35.0 * (t + 1))
            else:
                recs = ts.feed(dict(enumerate(frames)), now_ms=1.0e12 + 35.0 * (t + 1), width=W, height=H)
            for k in range(len(frames)):
                got = [{kk: v for kk, v in e.items() if kk != "time"} for e in log[k][marks[k]:]]
                check_events(got, want[k][t])
                if recs[k]["detection"] == "VJ":
                    p = pick(blob, frames[k])
                    assert (recs[k]["x"], recs[k]["y"], recs[k]["width"], recs[k]["height"],
                            recs[k]["confidence"]) == tuple(p[:5]), (k, t)
                    vj_seen += 1
        assert vj_seen >= len(frames)
    finally:
        c.close()


@pytest.mark.parametrize("K", [0, 1])
def test_track_init_from_detect_picks_from_the_callers_list(blob, K):
    """ht_track_init_from_detect keeps its meaning: the first maximum of the list it is given, here the K entries
    ht_detect copied out."""
    W, H = 320, 240
    frames = np.stack([crowd(n) for n in HANDOFF])
    c = context(W, H, len(frames), raw=BIG, K=K)
    try:
        rects, counts = c.detect_raw(frames, 5, 1)
        found = c.track_init_from_detect(frames, rects, counts, calc_angles=False)
        objs, wins = c.track(frames, n_calls=2)
        for i, name in enumerate(HANDOFF):
            g = oracle.detect(frames[i], blob, 5, 1, cap=BIG)[: c.K]
            ot = oracle_track(frames[i], g[first_max(g)], False, 2)
            assert found[i] == 1 and counts[i] == c.K, name
            assert_obj(objs[i], ot, name)
            assert wins[i] == ot.search_window(), name
    finally:
        c.close()
