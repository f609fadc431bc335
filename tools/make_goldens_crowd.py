#!/usr/bin/env python
"""Golden vectors of the grouping step and the VJ->CS hand-off on CROWDED frames, produced like tools/make_goldens.py
by executing the reference's own JavaScript (oracle/jsmini.py over the canvas shim) and asserting equality with the
C oracle on the way.

The existing goldens hold 1 to 3 faces per frame, so ccv.js's union-find (src/ccv.js:34-107) and the containment
filter have only been pinned on a handful of windows.  Each frame here (synth.crowd_frame, 320x240) has 200-450 raw
windows and 80-90 groups.  For each frame this records:

  * detect_objects(grayscale(canvas), cascade, 5, mn) for mn = 0, 1, 2, 3, 5;
  * facetrackr.js's VJ pass (a facetrackr.Tracker without whitebalancing, one track()): the TrackObj's x, y, width,
    height and confidence, i.e. the first maximum over the whole grouped list (src/facetrackr.js:157-165).

-> tests/golden/reference_js_crowd.json; replayed by tests/test_group_crowd_host.py (CPU).  The jobs run in parallel
processes; about 15 min on 8 cores (tree-walking interpreter).  Only runs where the reference sources exist.
"""
import json
import multiprocessing as mp
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))

import make_goldens as mg  # noqa: E402
import oracle  # noqa: E402
from headtrackr_b200 import synth  # noqa: E402
from oracle import jsmini  # noqa: E402

OUT = ROOT / "tests" / "golden" / "reference_js_crowd.json"
W, H, INTERVAL = 320, 240, 5
MIN_NEIGHBORS = (0, 1, 2, 3, 5)
FRAMES = [
    # name, crowd_frame(seed, W, H, side, pitch, jitter, variant)
    ("beyond_k", dict(seed=1, side=28, pitch=30, jitter=2, variant="grid")),   # first maximum at index 79
    ("tied_max", dict(seed=0, side=24, pitch=28, jitter=3, variant="grid")),   # the maximum is held by 4 groups
    ("two_sizes", dict(seed=0, side=24, pitch=28, jitter=2, variant="sizes")),
]


def make_frame(spec):
    return synth.crowd_frame(spec["seed"], W, H, spec["side"], spec["pitch"], spec["jitter"], spec["variant"])


def js_facetrackr_vj(it, frame):
    p = jsmini.JSObject()
    p.props.update(whitebalancing=False, calcAngles=False, sendEvents=False)
    trk = it.get(["headtrackr", "facetrackr", "Tracker"]).construct([p])
    it.call(trk.get("init"), trk, jsmini.CanvasShim(frame.copy()))
    it.call(trk.get("track"), trk)
    o = it.call(trk.get("getTrackingObject"), trk)
    return {k: o.get(k) for k in ("detection", "x", "y", "width", "height", "confidence")}


def job(args):
    name, mn = args
    it = mg.load_reference()
    frame = make_frame(dict(FRAMES)[name])
    t0 = time.time()
    if mn is None:
        it.run((mg.REF / "facetrackr.js").read_text())
        res = js_facetrackr_vj(it, frame)
    else:
        res, gray_sha = mg.js_detect(it, frame, INTERVAL, mn)
        assert gray_sha == mg.sha(oracle.grayscale(frame)), f"{name}: grayscale differs"
    print(f"{name} mn={mn}: {time.time() - t0:.0f}s", flush=True)
    return name, mn, res


def main():
    t_start = time.time()
    blob = synth.load_cascade_blob()
    jobs = [(name, mn) for name, _ in FRAMES for mn in MIN_NEIGHBORS + (None,)]
    with mp.Pool(min(len(jobs), mp.cpu_count())) as pool:
        results = pool.map(job, jobs, chunksize=1)
    by = {(name, mn): res for name, mn, res in results}
    gold = {"generator": "tools/make_goldens_crowd.py (reference JS executed by oracle/jsmini.py over the canvas shim)",
            "W": W, "H": H, "interval": INTERVAL, "frames": []}
    for name, spec in FRAMES:
        frame = make_frame(spec)
        lists = {}
        for mn in MIN_NEIGHBORS:
            rects = by[(name, mn)]
            want = [list(r) for r in oracle.detect(frame, blob, INTERVAL, mn)]
            assert rects == want, f"{name} mn={mn}: reference JS != C oracle"
            lists[str(mn)] = rects
        vj = by[(name, None)]
        g = lists["1"]
        best = max(range(len(g)), key=lambda i: (g[i][4], -i))
        assert vj["detection"] == "VJ"
        assert [vj["x"], vj["y"], vj["width"], vj["height"], vj["confidence"]] == g[best][:5], f"{name}: facetrackr pick"
        gold["frames"].append(dict(name=name, **spec, frame_sha256=mg.sha(frame), lists=lists, vj=vj))
        print(f"{name}: raw {len(lists['0'])}, groups {len(g)}, pick index {best}", flush=True)
    OUT.write_text(json.dumps(gold, indent=1))
    print(f"wrote {OUT} in {time.time() - t_start:.0f}s")


if __name__ == "__main__":
    main()
