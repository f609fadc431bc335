#!/usr/bin/env python
"""Generate tests/golden/reference_js_motion.json: the reference's own src/camshift.js, executed by oracle/jsmini.py
over the canvas shim, on the motion corpus of tests/test_track_motion_host.py (faces leaving the canvas, drifting left
and up, jumping, approaching and receding, re-entering; tracked rectangles partly or wholly outside the canvas).

Jobs (one camshift.Tracker each, initTracker on frame 0, then track() on every frame):
  * 160x120: every case with calcAngles on and off, one track() per frame, and three cases with three per frame;
  * 162x122 (W % 4 != 0): every case with calcAngles on.
The C oracle runs beside the JavaScript and must equal it on every call: x, y, width, height and the search window
exactly, the angle to 1e-12 (or both NaN).  Frames are stored as SHA-256 hashes, not pixels.

Only runs where /root/reference exists.  The jobs run in parallel processes: a few minutes on 8 cores.
"""
import json
import sys
import time
from multiprocessing import Pool
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

import oracle  # noqa: E402
import test_track_motion_host as mo  # noqa: E402
from oracle import jsmini  # noqa: E402

REF = Path("/root/reference/src")
OUT = mo.GOLD_PATH
THREE_CALLS = ("exit_left", "jump", "corner_init")


def jobs():
    out = [((160, 120), name, calc, 1) for name, _, _ in mo.CASES for calc in (False, True)]
    out += [((160, 120), name, False, 3) for name in THREE_CALLS]
    out += [((162, 122), name, True, 1) for name, _, _ in mo.CASES]
    return out


def same_angle(a, b):
    return (a != a and b != b) or a == b or abs(a - b) < 1e-12


def run_job(job):
    (W, H), name, calc, n_calls = job
    _, path, kind = mo.CASE[name]
    it = jsmini.Interpreter()
    it.run((REF / "camshift.js").read_text())
    Tracker = it.get(["headtrackr", "camshift", "Tracker"])
    Rectangle = it.get(["headtrackr", "camshift", "Rectangle"])
    params = jsmini.JSObject()
    params.props["calcAngles"] = bool(calc)
    trk = Tracker.construct([params])
    rect = mo.init_rect(kind, path, W, H)
    f0 = mo.frame(path, 0, W, H)
    it.call(trk.get("initTracker"), trk, jsmini.CanvasShim(f0.copy()), Rectangle.construct([float(v) for v in rect]))
    ot = oracle.CamshiftTracker(calc_angles=calc)
    ot.init_tracker(f0, *rect)
    frames = []
    for t in range(mo.T):
        f = mo.frame(path, t, W, H)
        canvas = jsmini.CanvasShim(f.copy())
        calls = []
        for c in range(n_calls):
            it.call(trk.get("track"), trk, canvas)
            o = jsmini.to_py(it.call(trk.get("getTrackObj"), trk))
            w = jsmini.to_py(it.call(trk.get("getSearchWindow"), trk))
            ot.track(f)
            oo = ot.track_obj()
            js_obj = [int(o["x"]), int(o["y"]), int(o["width"]), int(o["height"]), float(o["angle"])]
            js_win = [int(w["x"]), int(w["y"]), int(w["width"]), int(w["height"])]
            what = f"{name} {W}x{H} calc={calc} frame {t} call {c}"
            assert js_obj[:4] == [oo["x"], oo["y"], oo["width"], oo["height"]], f"{what}: {js_obj} vs {oo}"
            assert same_angle(js_obj[4], oo["angle"]), f"{what}: angle {js_obj[4]} vs {oo['angle']}"
            assert tuple(js_win) == ot.search_window(), f"{what}: window {js_win} vs {ot.search_window()}"
            calls.append(dict(obj=js_obj, window=js_win))
        frames.append(calls)
    return dict(name=name, path=path, rect_kind=kind, W=W, H=H, rect=list(rect), calc_angles=bool(calc),
                n_calls=n_calls, frames=frames)


def main():
    t0 = time.time()
    js = jobs()
    sizes = sorted({j[0] for j in js})
    gold = {"generator": "tools/make_goldens_motion.py (src/camshift.js executed by oracle/jsmini.py over the canvas "
                         "shim, on the corpus of tests/test_track_motion_host.py)",
            "reference": "auduno/headtrackr src/camshift.js", "T": mo.T,
            "frames": [dict(W=W, H=H, sha256={p: [mo.sha(mo.frame(p, t, W, H)) for t in range(mo.T)]
                                              for p in mo.PATHS}) for W, H in sizes],
            "cases": []}
    with Pool() as pool:
        for job, case in zip(js, pool.imap(run_job, js)):
            gold["cases"].append(case)
            print(f"{job}: JS == oracle ({time.time() - t0:.0f}s)", flush=True)
    OUT.write_text(json.dumps(gold, separators=(",", ":")) + "\n")
    print(f"wrote {OUT} in {time.time() - t0:.0f}s")


if __name__ == "__main__":
    main()
