"""GPU: k_cascade's table-driven paths with cascades other than the face model, bit-exact against the oracle run with
the same blob.

The corpus is synth.cascade_corpus() (tests/test_cascade_blobs_host.py checks the oracle against the reference's own
JavaScript on it): tie-prone tenths whose late-stage sums often equal their thresholds, 17-digit numbers (fp path),
1 to 9 stages (the n_groups == 1 emit block and the min(8, n_stages) group bound), odd feature shapes, the parser's
limits and the face model with one threshold moved by 1e-8.  Each test makes its own contexts and closes them.
"""
import sys
from functools import lru_cache
from pathlib import Path

import numpy as np
import pytest

import oracle
from headtrackr_b200 import Context, synth

sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tools"))
import pack_cascade  # noqa: E402

pytestmark = pytest.mark.gpu

BIG = 16384                  # list capacities that no frame here reaches
CORPUS = synth.cascade_corpus()
FP = {"fp", "limits_alpha", "limits_thr"} | {n for n in CORPUS if n.endswith("_fp")}


@lru_cache(maxsize=None)
def blob_of(name):
    kind, seed, kw = CORPUS[name]
    return pack_cascade.pack(synth.cascade(kind, seed, **kw))


def tup(d):
    return (d["x"], d["y"], d["width"], d["height"], d["confidence"], d.get("neighbors", d.get("neighbor")))


def context(W, H, n, blob, raw=BIG):
    return Context(max_width=W, max_height=H, max_frames=n, cascade=blob, max_raw_per_frame=raw, max_rects_per_frame=BIG)


def batch(blob, W, H, start=0):
    """7 frames, two quads: cascade faces, noise and a constant frame in the same quads"""
    f = lambda i: synth.frame(start + i, W, H, blob=blob)
    return np.stack([f(0), synth.frame(7, W, H, kind="noise"), f(1), synth.frame(0, W, H, kind="constant"), f(2),
                     synth.frame(8, W, H, kind="noise"), f(3)])


def check(c, blob, frames, interval, mns=(0, 1, 3)):
    raws = [oracle.detect(f, blob, interval, 0, cap=BIG) for f in frames]
    for mn in mns:
        got = c.detect(frames, interval, mn)
        assert c.last_warning is None, (interval, mn)
        if mn == 0:
            for i in range(len(frames)):
                r, cnt = c.debug_raw(i, cap=BIG)
                assert cnt == len(r) and r == raws[i], (interval, i)
        for i in range(len(frames)):
            want = raws[i] if mn == 0 else oracle.group(raws[i], mn, cap=BIG)
            assert [tup(d) for d in got[i]] == want, (interval, mn, i)
    return raws


# Every interval runs at two geometries.  The oracle's CPU time, not the GPU's, sets this file's duration: its
# grouping is quadratic in the raw list, which at 640x480 reaches 12,000 windows for the one- and two-stage cascades,
# so 640x480 runs the blobs with shorter lists (every path and group shape is in that subset).
GEOMETRIES = {(160, 120): (1, 2, 3, 5), (320, 240): (1, 3), (333, 251): (2, 5), (640, 480): (5,)}
VGA_BLOBS = ("ties", "fp", "shapes", "near_face", "short3", "short8_fp", "short9")


@pytest.mark.parametrize("W,H", list(GEOMETRIES))
def test_every_blob_equals_the_oracle(W, H):
    for name in CORPUS:
        if name.startswith("limits") and W * H > 100000:
            continue                                         # 2112 features evaluated lane by lane: small frames
        if W == 640 and name not in VGA_BLOBS:
            continue
        blob = blob_of(name)
        frames = batch(blob, W, H)
        c = context(W, H, len(frames), blob)
        try:
            for iv in GEOMETRIES[(W, H)]:
                raws = check(c, blob, frames, iv)
                assert raws[0] and raws[2], (name, iv)       # parity must not be vacuous
        finally:
            c.close()


VARIANTS = {"no_tma": {"HT_TMA": "0"}, "wave4_pipe": {"HT_WAVE": "4", "HT_DETECT_PIPE": "1"}, "late_ties": {},
            "no_late": {"HT_NO_LATE": "1"}}


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_blobs_through_the_variants(variant, monkeypatch):
    W, H = 320, 240
    for name in CORPUS:
        if variant == "no_late" and name in FP:
            continue                                         # already on the fp path
        if name.startswith("limits"):
            W, H = 160, 120
        blob = blob_of(name)
        frames = batch(blob, W, H, start=20)
        with monkeypatch.context() as m:
            for k, v in VARIANTS[variant].items():
                m.setenv(k, v)
            c = context(W, H, len(frames), blob)
            try:
                if variant == "late_ties":
                    c.debug_set_exactness(2)
                check(c, blob, frames, 5, mns=(0, 1))
            finally:
                c.close()


@pytest.mark.parametrize("W,H", [(1280, 720), (1920, 1080)])
def test_face_model_on_the_table_path_at_hd(blob, W, H, monkeypatch):
    monkeypatch.setenv("HT_NO_FAST", "1")
    frames = np.stack([synth.frame(i, W, H) for i in range(2)])
    c = context(W, H, 2, blob)
    try:
        raws = check(c, blob, frames, 5, mns=(0, 1))
        assert raws[0] and raws[1]
    finally:
        c.close()


def test_contexts_with_different_cascades_alternate(blob):
    """face, ties, face, fp, ties from one thread, device-resident batches: each context reloads its own cascade
    constants when another one was loaded in between; each result equals its own oracle."""
    import torch
    W, H = 320, 240
    blobs = {"face": blob, "ties": blob_of("ties"), "fp": blob_of("fp")}
    ctxs = {k: context(W, H, 7, b) for k, b in blobs.items()}
    try:
        frames = {k: batch(b, W, H, start=40) for k, b in blobs.items()}
        dev = {k: torch.from_numpy(f).cuda() for k, f in frames.items()}
        torch.cuda.synchronize()
        for k in ("face", "ties", "face", "fp", "ties"):
            got = ctxs[k].detect(dev[k], 5, 1)
            for i in range(7):
                assert [tup(d) for d in got[i]] == oracle.detect(frames[k][i], blobs[k], 5, 1), (k, i)
    finally:
        for c in ctxs.values():
            c.close()


def first_max(g):
    return max(range(len(g)), key=lambda i: (g[i][4], -i))


@pytest.mark.parametrize("mode", ["unpipelined", "pipelined", "stream_step"])
def test_handoff_with_the_ties_cascade(mode):
    import torch
    W, H = 320, 240
    b = blob_of("ties")
    frames = np.stack([synth.frame(60 + i, W, H, blob=b) for i in range(4)] + [synth.frame(0, W, H, kind="constant")])
    n = len(frames)
    c = Context(max_width=W, max_height=H, max_frames=n, cascade=b, max_raw_per_frame=BIG)
    try:
        if mode == "stream_step":
            c.stream_reset()
            ev = c.stream_step(frames)
            for i in range(n):
                g = oracle.detect(frames[i], b, 5, 1)
                assert ev[i]["detection"] == "VJ" and ev[i]["found"] == bool(g), i
                if g:
                    p = g[first_max(g)]
                    assert (ev[i]["x"], ev[i]["y"], ev[i]["width"], ev[i]["height"], ev[i]["confidence"]) == tuple(p[:5])
            return
        if mode == "unpipelined":
            _, found, objs, _ = c.detect_track(frames, 5, 1, calc_angles=False, n_calls=3)
        else:
            c.set_pipeline(True)
            dev = torch.from_numpy(frames).cuda()
            outs = (torch.zeros((n, c.K, 6), dtype=torch.float64, device="cuda"),
                    torch.zeros((n,), dtype=torch.int32, device="cuda"), torch.zeros((n,), dtype=torch.int32, device="cuda"),
                    torch.zeros((n, 6), dtype=torch.int32, device="cuda"), torch.zeros((n, 4), dtype=torch.int32, device="cuda"))
            torch.cuda.synchronize()
            for _ in range(2):
                c.detect_track(dev, 5, 1, calc_angles=False, n_calls=3, outputs=outs)
            c.sync()
            found = outs[2].cpu().tolist()
            objs = [dict(x=int(r[0]), y=int(r[1]), width=int(r[2]), height=int(r[3])) for r in outs[3].cpu().numpy()]
        n_found = 0
        for i in range(n):
            _, fo, obj = oracle.detect_track(frames[i], b, 5, 1, False, 3)
            assert found[i] == fo, i
            if fo:
                n_found += 1
                assert tuple(objs[i][k] for k in ("x", "y", "width", "height")) == \
                    tuple(obj[k] for k in ("x", "y", "width", "height")), i
        assert n_found >= 3
    finally:
        c.close()
