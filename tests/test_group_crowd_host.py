"""The grouping step and facetrackr's VJ->CS pick on crowded frames (synth.crowd_frame), on the CPU.

Frames with 1 to 3 faces give 2 to 5 groups, so they never run the parts of the grouping step that depend on long lists:
class order over many components, ties for the maximum confidence, the containment filter at min_neighbors >= 3, and
lists longer than the device's 32-entry ballot blocks or its default capacities.  This file

  * re-checks the C oracle against tests/golden/reference_js_crowd.json (tools/make_goldens_crowd.py: the reference's
    own ccv.js and facetrackr.js executed on three 320x240 crowds);
  * checks that CROWD, the corpus tests/test_gpu_crowd.py runs on the device, has the properties those tests rely on,
    so that they cannot pass vacuously.
"""
import hashlib
import json
from pathlib import Path

import numpy as np
import pytest

import oracle
from headtrackr_b200 import synth

GOLD = json.loads((Path(__file__).resolve().parent / "golden" / "reference_js_crowd.json").read_text())

# name -> (W, H, crowd_frame keyword arguments)
CROWD = {
    "beyond_k": (320, 240, dict(seed=1, side=28, pitch=30, jitter=2)),          # first maximum at index 79 (> 63)
    "tied_max": (320, 240, dict(seed=0, side=24, pitch=28, jitter=3)),          # the maximum is shared
    "grid_ties": (320, 240, dict(seed=0, side=24, pitch=24, jitter=0)),         # every group ties at the maximum
    "two_sizes": (320, 240, dict(seed=0, side=24, pitch=28, jitter=2, variant="sizes")),
    "nested": (320, 240, dict(seed=0, side=24, pitch=28, jitter=2, variant="nested")),
    "edges": (320, 240, dict(seed=0, side=24, pitch=28, jitter=2, variant="edges")),
    "chains": (320, 240, dict(seed=0, side=24, pitch=28, variant="chains")),
    "small": (160, 120, dict(seed=2, side=24, pitch=26, jitter=2)),
    "vga": (640, 480, dict(seed=0, side=28, pitch=30, jitter=2)),               # raw list above 1024
    "hd": (1280, 720, dict(seed=3, side=32, pitch=34, jitter=2)),
}


def crowd(name):
    W, H, kw = CROWD[name]
    return synth.crowd_frame(W=W, H=H, **kw)


def first_max(lst):
    """src/facetrackr.js:157-165: the first entry of greatest confidence (-1 for an empty list)"""
    best = -1
    for i, r in enumerate(lst):
        if best < 0 or r[4] > lst[best][4]:
            best = i
    return best


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


@pytest.mark.parametrize("case", GOLD["frames"], ids=lambda c: c["name"])
def test_oracle_equals_reference_js_on_crowds(case, blob):
    spec = {k: case[k] for k in ("seed", "side", "pitch", "jitter", "variant")}
    f = synth.crowd_frame(W=GOLD["W"], H=GOLD["H"], **spec)
    assert sha(f) == case["frame_sha256"]                   # the generator still makes the frame the goldens were cut from
    raw = oracle.detect(f, blob, GOLD["interval"], 0)
    for mn, want in case["lists"].items():
        got = oracle.detect(f, blob, GOLD["interval"], int(mn))
        assert [list(r) for r in got] == want, mn
        if int(mn) > 0:                                     # the grouping alone, from the raw list
            assert [list(r) for r in oracle.group(raw, int(mn))] == want, mn
    g = case["lists"]["1"]
    b = first_max(g)
    vj = case["vj"]
    assert [vj["x"], vj["y"], vj["width"], vj["height"], vj["confidence"]] == g[b][:5]
    # the oracle's own detect -> pick -> initTracker seeds the same face
    _, found, _ = oracle.detect_track(f, blob, GOLD["interval"], 1, n_calls=0)
    assert found == 1


def test_golden_crowds_cover_the_pick_and_ties():
    by = {c["name"]: c for c in GOLD["frames"]}
    g = by["beyond_k"]["lists"]["1"]
    assert first_max(g) > 63 and len(g) >= 64
    g = by["tied_max"]["lists"]["1"]
    top = max(r[4] for r in g)
    assert sum(r[4] == top for r in g) >= 2
    for c in GOLD["frames"]:
        assert len(c["lists"]["3"]) > 0 and len(c["lists"]["0"]) > len(c["lists"]["1"])


@pytest.fixture(scope="module")
def corpus(blob):
    """name -> (raw list, grouped list at min_neighbors 1, 3, 5) from the oracle at interval 5"""
    out = {}
    for name in CROWD:
        f = crowd(name)
        g1, raw = oracle.detect(f, blob, 5, 1, want_raw=True)
        out[name] = dict(raw=raw, g1=g1, g3=oracle.group(raw, 3), g5=oracle.group(raw, 5))
        assert g1 == oracle.group(raw, 1)
    return out


def test_corpus_properties(corpus):
    """What tests/test_gpu_crowd.py needs from CROWD: at least 64 groups, a first maximum past index 63 (the default
    max_rects_per_frame), a tie for the maximum, a raw list above 1024 (the default max_raw_per_frame), 33 or more kept
    rectangles (so classes too: k_group's steps 3 and 4 run more than one 32-entry ballot block), and non-empty lists
    at min_neighbors 3 and 5."""
    g = {k: v["g1"] for k, v in corpus.items()}
    assert max(len(v) for v in g.values()) >= 64
    assert first_max(g["beyond_k"]) > 63
    for name in ("tied_max", "grid_ties"):
        top = max(r[4] for r in g[name])
        assert sum(r[4] == top for r in g[name]) >= 2, name
    assert len(corpus["vga"]["raw"]) > 1024
    assert len(corpus["hd"]["raw"]) > 1024
    assert sum(len(v) >= 33 for v in g.values()) >= 5
    assert all(len(v["g3"]) > 0 for v in corpus.values() if len(v["g1"]) >= 33)
    assert sum(len(v["g5"]) > 0 for v in corpus.values()) >= 5
    # the variants do what their names say
    assert len({r[2] for r in corpus["two_sizes"]["raw"]}) >= 2
    W, H, _ = CROWD["edges"]
    assert any(r[0] + r[2] > W - 12 for r in g["edges"]) and any(r[1] + r[3] > H - 12 for r in g["edges"])
    assert any(r[2] >= 72 for r in g["nested"])            # the large face around the small one is found
