#!/usr/bin/env python
"""Golden vectors of detection with OTHER cascades than the face model, produced like tools/make_goldens_crowd.py by
executing the reference's own JavaScript (oracle/jsmini.py over the canvas shim) and asserting equality with the C
oracle on the way.

src/ccv.js's detect_objects takes the cascade as an argument; every test before this one passed it the face model.
Here each cascade of synth.cascade_corpus() (tie-prone tenths, 17-digit fp numbers, 1 to 9 stages, odd feature
shapes, the parser's limits, the face model with one threshold moved by 1e-8) is passed as a JS object literal, on
frames carrying faces voted from that cascade's own points (synth.frame(..., blob=b)).  For each cascade this records
detect_objects(grayscale(canvas), cascade, interval, mn) for 160x120 and 171x133 frames, intervals 5 and 2 and
mn = 0 and 1; the three limits cascades (2112 features each) run on the 160x120 frame at interval 5 only.

-> tests/golden/reference_js_cascades.json, replayed by tests/test_cascade_blobs_host.py.  To keep it small:
  * each cascade is embedded as its HTC1 blob (tools/pack_cascade.py), zlib-compressed and base64-encoded; near_face
    as the stage and threshold it changes in the face model's blob (checked by its SHA-256);
  * the grouped lists (mn = 1) are stored whole, the raw lists (mn = 0, up to 800 windows) as their length and the
    SHA-256 of their canonical JSON (rects_digest).
The jobs run in parallel processes (tree-walking interpreter).  Only runs where the reference sources exist.
"""
import base64
import hashlib
import json
import multiprocessing as mp
import sys
import struct
import time
import zlib
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))

import make_goldens as mg  # noqa: E402
import oracle  # noqa: E402
import pack_cascade  # noqa: E402
from headtrackr_b200 import synth  # noqa: E402
from oracle import jsmini  # noqa: E402

OUT = ROOT / "tests" / "golden" / "reference_js_cascades.json"
FRAMES = ((160, 120, 0), (171, 133, 1))     # W, H, synth.frame index
INTERVALS = (5, 2)
MIN_NEIGHBORS = (0, 1)


def rects_digest(rects):
    """SHA-256 of a detection list's canonical JSON: [x, y, width, height, confidence, neighbors] per entry"""
    canon = [[float(v) for v in r[:5]] + [int(r[5])] for r in rects]
    return hashlib.sha256(json.dumps(canon, separators=(",", ":")).encode()).hexdigest()


def encode_cascade(name, blob, face_blob):
    """A golden cascade entry: near_face as the one stage threshold it changes in the face model's blob, any other
    cascade as its whole blob"""
    if name != "near_face":
        return dict(blob_zlib_b64=base64.b64encode(zlib.compress(blob, 9)).decode())
    n_stages = struct.unpack_from("<I", blob, 4)[0]
    j = next(j for j in range(n_stages) if blob[24 + 16 * j: 40 + 16 * j] != face_blob[24 + 16 * j: 40 + 16 * j])
    entry = dict(face_sha256=hashlib.sha256(face_blob).hexdigest(), stage=j,
                 threshold=struct.unpack_from("<d", blob, 32 + 16 * j)[0])
    assert decode_cascade(entry, face_blob) == blob
    return entry


def decode_cascade(entry, face_blob):
    """The HTC1 blob of a golden cascade entry"""
    if "blob_zlib_b64" in entry:
        return zlib.decompress(base64.b64decode(entry["blob_zlib_b64"]))
    assert hashlib.sha256(face_blob).hexdigest() == entry["face_sha256"]
    b = bytearray(face_blob)
    struct.pack_into("<d", b, 32 + 16 * entry["stage"], entry["threshold"])
    return bytes(b)


def cases(name):
    small = name.startswith("limits")
    for W, H, idx in FRAMES[:1] if small else FRAMES:
        for interval in INTERVALS[:1] if small else INTERVALS:
            yield W, H, idx, interval


def make_cascade(name):
    kind, seed, kw = synth.cascade_corpus()[name]
    return synth.cascade(kind, seed, **kw)


def js_detect(it, frame, cascade_js, interval, mn):
    canvas = jsmini.CanvasShim(frame.copy())
    gray = it.call(it.get(["headtrackr", "ccv", "grayscale"]), jsmini.undefined, canvas)
    res = it.call(it.get(["headtrackr", "ccv", "detect_objects"]), jsmini.undefined, gray, cascade_js, float(interval),
                  float(mn))
    out = []
    for r in jsmini.to_py(res):
        nb = r.get("neighbors", r.get("neighbor"))
        out.append([r["x"], r["y"], r["width"], r["height"], r["confidence"], int(nb)])
    return out, mg.sha(canvas.pix[..., 0])


def job(args):
    name, W, H, idx, interval, mn = args
    it = mg.load_reference()
    c = make_cascade(name)
    it.run("var synth_cascade = " + json.dumps(c) + ";")
    frame = synth.frame(idx, W, H, blob=pack_cascade.pack(c))
    t0 = time.time()
    res, gray_sha = js_detect(it, frame, it.get(["synth_cascade"]), interval, mn)
    assert gray_sha == mg.sha(oracle.grayscale(frame)), f"{name}: grayscale differs"
    print(f"{name} {W}x{H} i={interval} mn={mn}: {len(res)} rects, {time.time() - t0:.0f}s", flush=True)
    return args, res


def main():
    t_start = time.time()
    names = list(synth.cascade_corpus())
    jobs = [(name, W, H, idx, interval, mn) for name in names for W, H, idx, interval in cases(name) for mn in MIN_NEIGHBORS]
    jobs.sort(key=lambda j: not j[0].startswith("limits"))          # the slowest first
    with mp.Pool(mp.cpu_count()) as pool:
        results = dict(pool.map(job, jobs, chunksize=1))
    gold = {"generator": "tools/make_goldens_cascades.py (reference JS executed by oracle/jsmini.py over the canvas "
                         "shim, each cascade passed to detect_objects as an object literal)", "cascades": []}
    face_blob = synth.load_cascade_blob()
    for name in names:
        c = make_cascade(name)
        blob = pack_cascade.pack(c)
        runs = []
        for W, H, idx, interval in cases(name):
            frame = synth.frame(idx, W, H, blob=blob)
            lists = {}
            for mn in MIN_NEIGHBORS:
                rects = results[(name, W, H, idx, interval, mn)]
                want = [list(r) for r in oracle.detect(frame, blob, interval, mn)]
                assert rects == want, f"{name} {W}x{H} i={interval} mn={mn}: reference JS != C oracle"
                lists[str(mn)] = rects if mn else dict(n=len(rects), sha256=rects_digest(rects))
            runs.append(dict(W=W, H=H, index=idx, interval=interval, frame_sha256=mg.sha(frame), lists=lists))
        gold["cascades"].append(dict(name=name, **encode_cascade(name, blob, face_blob), runs=runs))
    entries = ",\n".join(json.dumps(e, separators=(",", ":")) for e in gold["cascades"])   # one cascade per line
    OUT.write_text('{"generator": ' + json.dumps(gold["generator"]) + ', "cascades": [\n' + entries + "\n]}\n")
    print(f"wrote {OUT} in {time.time() - t_start:.0f}s")


if __name__ == "__main__":
    main()
