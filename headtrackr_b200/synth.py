"""Deterministic synthetic RGBA frames for tests and bench (integer-only, so every machine agrees).

The reference ships no sample images (SURVEY.md §4).  Noise alone yields zero detections, which
would make parity vacuous, so frames carry "faces" synthesised from the cascade itself
(SURVEY.md Appendix A1): a 24x24 template whose pixels are the +-alpha votes of every feature
point of `headtrackr.cascade` (/root/reference/src/cascade.js:19), resized and pasted with a
skin-like tint on a blurred-noise background.

frame(i) is a pure function of (seed_base + i, W, H): PCG64 integers + integer box blurs +
the canvas-shim bilinear resize (same definition as oracle/ht_oracle.h).
"""
import copy
import struct
from functools import lru_cache
from math import factorial
from pathlib import Path
from statistics import NormalDist

import numpy as np

DATA = Path(__file__).resolve().parent / "data" / "cascade_face.bin"
SEED_BASE = 0xB200


def load_cascade_blob(path=DATA):
    return Path(path).read_bytes()


def parse_blob(blob):
    assert blob[:4] == b"HTC1"
    n_stages, n_feat, w, h, _ = struct.unpack_from("<5I", blob, 4)
    stages = [struct.unpack_from("<IId", blob, 24 + 16 * j) for j in range(n_stages)]
    fo = 24 + 16 * n_stages
    ao = fo + 32 * n_feat
    feats = []
    for k in range(n_feat):
        rec = blob[fo + 32 * k: fo + 32 * k + 32]
        size = rec[0]
        sb = lambda v: v - 256 if v > 127 else v
        p = [(sb(rec[2 + q]), rec[7 + q], rec[12 + q]) for q in range(5)]
        n = [(sb(rec[17 + q]), rec[22 + q], rec[27 + q]) for q in range(5)]
        a_fail, a_pass = struct.unpack_from("<dd", blob, ao + 16 * k)
        feats.append(dict(size=size, p=p, n=n, a_fail=a_fail, a_pass=a_pass))
    return dict(n_stages=n_stages, n_features=n_feat, width=w, height=h, stages=stages, features=feats)


@lru_cache(maxsize=2)
def face_template(blob=None):
    """24x24 u8 template voted by the cascade's own feature points (pure-Python fp64, deterministic)."""
    c = parse_blob(blob if blob is not None else load_cascade_blob())
    n = c["width"]
    vote = [[0.0] * n for _ in range(n)]
    for f in c["features"]:
        for pts, sign in ((f["p"], 1.0), (f["n"], -1.0)):
            for (z, x, y) in pts[: f["size"]]:
                if z < 0:
                    continue
                s = 1 << z
                v = sign * f["a_pass"] / float(4 ** z)
                for yy in range(y * s, (y + 1) * s):
                    for xx in range(x * s, (x + 1) * s):
                        vote[yy][xx] += v
    lo = min(min(r) for r in vote)
    hi = max(max(r) for r in vote)
    t = np.zeros((n, n), np.uint8)
    for y in range(n):
        for x in range(n):
            t[y, x] = int((vote[y][x] - lo) * 255.0 / (hi - lo) + 0.5)
    return t


def shim_resize(src, dw, dh, sx=0, sy=0, sw=None, sh=None):
    """Canvas-shim drawImage (see oracle/ht_oracle.h) vectorised in numpy int64. src: (H,W) u8."""
    src = np.asarray(src)
    if sw is None:
        sw = src.shape[1] - sx
    if sh is None:
        sh = src.shape[0] - sy
    X = np.arange(dw, dtype=np.int64)
    Y = np.arange(dh, dtype=np.int64)
    un = (2 * X + 1) * sw - dw
    vn = (2 * Y + 1) * sh - dh
    x0 = np.floor_divide(un, 2 * dw)
    y0 = np.floor_divide(vn, 2 * dh)
    fx = un - x0 * 2 * dw
    fy = vn - y0 * 2 * dh
    xa = np.clip(x0, 0, sw - 1) + sx
    xb = np.clip(x0 + 1, 0, sw - 1) + sx
    ya = np.clip(y0, 0, sh - 1) + sy
    yb = np.clip(y0 + 1, 0, sh - 1) + sy
    s = src.astype(np.int64)
    Dx, Dy = 2 * dw, 2 * dh
    wx0 = (Dx - fx)[None, :]
    wx1 = fx[None, :]
    wy0 = (Dy - fy)[:, None]
    wy1 = fy[:, None]
    num = (wx0 * wy0 * s[ya][:, xa] + wx1 * wy0 * s[ya][:, xb] +
           wx0 * wy1 * s[yb][:, xa] + wx1 * wy1 * s[yb][:, xb])
    return ((num + 2 * dw * dh) // (4 * dw * dh)).astype(np.uint8)


def _box_blur(a, radius, passes):
    """Integer box blur with edge replication on the last two axes of an (H,W,C) int32 array."""
    k = 2 * radius + 1
    for _ in range(passes):
        for axis in (0, 1):
            pad = [(0, 0)] * a.ndim
            pad[axis] = (radius + 1, radius)
            p = np.pad(a, pad, mode="edge")
            c = np.cumsum(p, axis=axis, dtype=np.int64)
            hi = np.take(c, np.arange(k, k + a.shape[axis]), axis=axis)
            lo = np.take(c, np.arange(0, a.shape[axis]), axis=axis)
            a = ((hi - lo + k // 2) // k).astype(np.int32)
    return a


def frame(index, W=640, H=480, n_faces=None, seed_base=SEED_BASE, kind="faces", blob=None, return_faces=False):
    """RGBA u8 (H,W,4) frame.  kind: 'faces' | 'noise' | 'constant' | 'gradient'."""
    rng = np.random.Generator(np.random.PCG64(seed_base + int(index)))
    out = np.empty((H, W, 4), np.uint8)
    out[..., 3] = 255
    faces = []
    if kind == "constant":
        out[..., :3] = 128
    elif kind == "gradient":
        out[..., :3] = ((np.arange(W, dtype=np.int64) * 255) // max(W - 1, 1)).astype(np.uint8)[None, :, None]
    else:
        noise = rng.integers(0, 256, size=(H, W, 3), dtype=np.int64).astype(np.int32)
        if kind == "noise":
            out[..., :3] = noise.astype(np.uint8)
        else:
            b = _box_blur(noise, 2, 2)
            lo = b.min(axis=(0, 1), keepdims=True)
            hi = b.max(axis=(0, 1), keepdims=True)
            b = ((b - lo) * 255) // np.maximum(hi - lo, 1)
            out[..., :3] = b.astype(np.uint8)
            tmpl = face_template(blob)
            if n_faces is None:
                n_faces = int(rng.integers(1, 4))
            max_side = max(28, int(0.4 * H))
            for _ in range(n_faces):
                side = int(rng.integers(28, max_side + 1))
                x = int(rng.integers(0, W - side + 1))
                y = int(rng.integers(0, H - side + 1))
                t = shim_resize(tmpl, side, side).astype(np.int32)
                out[y:y + side, x:x + side, 0] = t.astype(np.uint8)
                out[y:y + side, x:x + side, 1] = ((t * 200) >> 8).astype(np.uint8)
                out[y:y + side, x:x + side, 2] = ((t * 150) >> 8).astype(np.uint8)
                faces.append((x, y, side))
    return (out, faces) if return_faces else out


def _paste_face(out, x, y, side, blob=None):
    """The face template resized to side x side with frame()'s tint, clipped to the frame at its right and bottom."""
    H, W = out.shape[:2]
    t = shim_resize(face_template(blob), side, side).astype(np.int32)[: H - y, : W - x]
    h, w = t.shape
    out[y:y + h, x:x + w, 0] = t.astype(np.uint8)
    out[y:y + h, x:x + w, 1] = ((t * 200) >> 8).astype(np.uint8)
    out[y:y + h, x:x + w, 2] = ((t * 150) >> 8).astype(np.uint8)


def crowd_frame(seed, W=320, H=240, side=24, pitch=None, jitter=0, variant="grid", blob=None):
    """A frame crowded with faces, for the grouping step: many raw windows and many groups.

    The background is frame(seed, W, H, n_faces=0).  Faces of `side` px are pasted on a grid of `pitch` px from (0,0),
    each cell shifted by rng.integers(0, jitter + 1) in x and in y (rng = default_rng(seed)) and clamped to the frame.
    variant:
      grid     the grid alone
      sizes    rows alternate between side and side * 3 // 2 (two face sizes in one frame)
      nested   the grid, then one face of 4 * side at the frame's centre with a face of side px inside it
               (the containment filter of the grouping step)
      edges    the grid shifted so that the last column and row are cut by the right and bottom edges
      chains   rows of overlapping faces spaced by 2 * floor(side / 4 + 0.5) + {0, 1} px: the windows of neighbouring
               faces lie near the grouping predicate's distance floor(w / 4 + 0.5) of each other
    Integer-only, like frame()."""
    pitch = side if pitch is None else pitch
    rng = np.random.default_rng(seed)
    out = frame(seed, W, H, n_faces=0, blob=blob)
    if variant == "chains":
        d = (side + 2) // 4                                # floor(side / 4 + 0.5)
        for y in range(0, H - side + 1, pitch):
            x = 0
            while x + side <= W:
                _paste_face(out, x, y, side, blob)
                x += 2 * d + int(rng.integers(0, 2))
        return out
    off = (side // 2) if variant == "edges" else 0
    for row, y0 in enumerate(range(off, H - (0 if variant == "edges" else side) + 1, pitch)):
        s = side * 3 // 2 if (variant == "sizes" and row % 2) else side
        for x0 in range(off, W - (0 if variant == "edges" else s) + 1, pitch):
            x = min(x0 + int(rng.integers(0, jitter + 1)), W - (1 if variant == "edges" else s))
            y = min(y0 + int(rng.integers(0, jitter + 1)), H - (1 if variant == "edges" else s))
            _paste_face(out, x, y, s, blob)
    if variant == "nested":
        big = 4 * side
        x, y = max(0, (W - big) // 2), max(0, (H - big) // 2)
        _paste_face(out, x, y, big, blob)
        _paste_face(out, x + big // 4, y + big // 4, side, blob)
    return out


def batch(n, W=640, H=480, start=0, **kw):
    return np.stack([frame(start + i, W, H, **kw) for i in range(n)])


# ---- synthetic cascades: other models than the face one, for the table-driven paths of the cascade kernel ----
# cascade(kind, seed) returns a cascade in the schema of src/cascade.js (tools/pack_cascade.pack turns it into a blob).
# Numbers are built from integers and decimal literals only, so every machine builds the same model.
LIMIT_ALPHA, LIMIT_THR = "21.47483647", "10995.11627775"   # largest |alpha| and |threshold| of the integer-table path


def _dec(n, digits):
    """The decimal literal n * 10^-digits as a float (float() of the literal, like JS Number())."""
    s = "-" if n < 0 else ""
    n = abs(n)
    return float(f"{s}{n // 10 ** digits}.{n % 10 ** digits:0{digits}d}")


def _feature(rng, size, holes=True):
    f = {"size": size}
    for side in "pn":
        zs, xs, ys = [], [], []
        for q in range(size):
            z = int(rng.integers(0, 3))
            if q and holes and int(rng.integers(0, 4)) == 0:
                z = -1
            lim = (24 >> max(z, 0)) - 1
            zs.append(z)
            xs.append(int(rng.integers(0, lim + 1)) if z >= 0 else 0)
            ys.append(int(rng.integers(0, lim + 1)) if z >= 0 else 0)
        f[side + "z"], f[side + "x"], f[side + "y"] = zs, xs, ys
    return f


def _stage(feats, alphas, thr):
    """alphas: alpha_pass of each feature (alpha[2k] = -alpha[2k+1], the only form the library accepts)."""
    return {"count": len(feats), "threshold": thr, "feature": feats,
            "alpha": [v for a in alphas for v in (-a, a)]}


def _model(stages):
    return {"count": len(stages), "width": 24, "height": 24, "stage_classifier": stages}


def _fire_probability(f):
    """P(min(p) > max(n)) when the valid points read independent, identically distributed pixels."""
    k_p = sum(1 for z in f["pz"] if z >= 0)
    k_n = sum(1 for z in f["nz"] if z >= 0)
    return factorial(k_p) * factorial(k_n) / factorial(k_p + k_n)


def _grid_stage(rng, n, spread, digits, grid_alphas=None, max_size=3, tie=None):
    """n features; alphas from grid_alphas (tenths) or random `digits`-digit decimals in (0.05, 1).  The threshold lies
    `spread` standard deviations below the stage sum's mean on i.i.d. pixels, rounded down to the grid of the alphas
    (0.1 or 10^-digits): early stages pass most windows, late ones about half.  With `tie`, the threshold is chosen
    for exact ties instead (None when the draw allows none)."""
    feats = [_feature(rng, int(rng.integers(1, max_size + 1))) for _ in range(n)]
    if grid_alphas is not None:
        units = [int(rng.choice(grid_alphas)) for _ in range(n)]
        unit_digits = 1
    else:
        units = [int(rng.integers(5 * 10 ** (digits - 2), 10 ** digits)) for _ in range(n)]
        unit_digits = digits
    units = [-u if int(rng.integers(0, 8)) == 0 else u for u in units]   # a few features vote against the face
    alphas = [_dec(u, unit_digits) for u in units]
    ps = [_fire_probability(f) for f in feats]
    mean = sum(u * (2 * p - 1) for u, p in zip(units, ps))
    std = sum(4 * u * u * p * (1 - p) for u, p in zip(units, ps)) ** 0.5
    t = int(np.floor(mean - spread * std))
    if tie is not None:
        # among the thresholds that pass at least 30 % of the windows (fire patterns weighted with ps), the one with the
        # most probable patterns whose exact sum equals it and whose ordered fp64 sum the reference passes
        # (tie="pass") or fails (tie="fail")
        pats = []
        for bits in range(1 << n):
            exact, fp, w = 0, 0.0, 1.0
            for k in range(n):
                on = (bits >> k) & 1
                exact += units[k] if on else -units[k]
                fp += alphas[k] if on else -alphas[k]
                w *= ps[k] if on else 1.0 - ps[k]
            pats.append((exact, fp, w))
        best = (-1.0, 0)
        for tt in sorted({e for e, _, _ in pats}):
            thr = _dec(tt, unit_digits)
            p_pass = sum(w for _, fp, w in pats if not (fp < thr))
            p_tie = sum(w for e, fp, w in pats if e == tt and (not (fp < thr)) == (tie == "pass"))
            if 0.3 <= p_pass <= 0.75 and p_tie > best[0]:
                best = (p_tie, tt)
        if best[0] < 0.05:
            return None                                      # no such threshold: the caller draws another stage
        t = best[1]
    return _stage(feats, alphas, _dec(t, unit_digits))


def cascade(kind, seed=0, n_stages=None, fp=False):
    """A synthetic cascade (src/cascade.js schema).  kind:
      ties       14 stages, alphas from {0.1, 0.2, 0.3, 0.6, 0.7}, thresholds on the same 0.1 grid: exact decimal
                 stage sums often equal the threshold, in the late stages (>= 8) too, where the fp64 verdict goes
                 both ways (0.1 + 0.2 >= 0.3 passes, -0.1 - 0.2 < -0.3 fails)
      fp         the same structure with 17-digit alphas and thresholds (not 8-digit decimals) and a last stage of
                 120 features
      short      n_stages in 1..9 stages, 8-digit decimals (integer-table path) or, with fp=True, 17-digit ones
      shapes     feature sizes 1-5, unused slots 1-4 on both sides, points at 0 and at the last coordinate of each
                 level, a feature whose p and n point coincide, alpha +-0.0, zero-feature stages with thresholds
                 <= 0, late stages of 1, 32 and 33 features
      limits     64 stages (four distinct ones, repeated) and 2112 features with one alpha of 21.47483647 and one
                 threshold of -10995.11627775;
                 n_stages=1 / 2 moves that alpha / threshold one unit of 1e-8 past the integer limit
      near_face  the face model with stage 8's threshold raised by 1e-8"""
    rng = np.random.default_rng(seed)
    if kind == "ties":
        stages = []
        for j in range(14):
            n = int(rng.integers(2, 5)) if j < 8 else int(rng.integers(3, 6))
            tie = None if j < 8 else ("pass", "fail")[j % 2]
            st = None
            while st is None:
                st = _grid_stage(rng, n, 1.0, 1, grid_alphas=(1, 2, 3, 6, 7), tie=tie)
            stages.append(st)
        return _model(stages)
    if kind == "fp":
        stages = [_grid_stage(rng, int(rng.integers(2, 6)), 1.2 if j < 8 else 0.3, 17) for j in range(11)]
        stages.append(_grid_stage(rng, 120, 0.5, 17))
        return _model(stages)
    if kind == "short":
        spread = NormalDist().inv_cdf(0.02 ** (1 / n_stages))   # about 2 % of the windows pass all stages
        return _model([_grid_stage(rng, int(rng.integers(2, 6)), spread, 17 if fp else 8) for _ in range(n_stages)])
    if kind == "shapes":
        stages = []
        for j in range(12):
            n = {8: 1, 9: 32, 11: 33}.get(j, int(rng.integers(3, 7)))
            st = _grid_stage(rng, n, 0.7, 8, max_size=5)
            stages.append(st)
        edge = stages[0]["feature"]
        for k, z in enumerate((0, 1, 2)):                  # points at 0 and at the last coordinate of each level
            lim = (24 >> z) - 1
            edge[k % len(edge)].update(pz=[z, z], px=[0, lim], py=[lim, 0], nz=[z, -1], nx=[lim, 0], ny=[lim, 0], size=2)
        for size in range(1, 6):                           # every size, with unused slots 1..4 on both sides
            f = _feature(rng, size, holes=False)
            for side in "pn":
                if size > 1:
                    f[side + "z"][size - 1] = -1
                    f[side + "x"][size - 1] = f[side + "y"][size - 1] = 0
            stages[1 + size % 4]["feature"].append(f)
            stages[1 + size % 4]["alpha"] += [-0.25, 0.25]
        same = {"size": 1, "pz": [1], "px": [5], "py": [7], "nz": [1], "nx": [5], "ny": [7]}   # never fires
        stages[3]["feature"].append(same)
        stages[3]["alpha"] += [-0.125, 0.125]
        stages[10]["feature"].append(dict(same, pz=[2], px=[3], py=[4], nz=[2], nx=[3], ny=[4]))
        stages[10]["alpha"] += [-0.0, 0.0]                 # alpha +-0.0 in both orders
        stages[10]["feature"].append(_feature(rng, 2))
        stages[10]["alpha"] += [0.0, -0.0]
        stages.insert(5, _stage([], [], 0.0))              # zero-feature stages: in a lane-per-window group and late
        stages.insert(11, _stage([], [], 0.0))
        stages.insert(12, _stage([], [], -0.5))
        for st in stages:
            st["count"] = len(st["feature"])
        return _model(stages)
    if kind == "limits":
        spread = NormalDist().inv_cdf(0.02 ** 0.25)        # a window passes all 64 stages when it passes the four
        protos = [_grid_stage(rng, 33, spread, 8) for _ in range(4)]   # 2112 features: four stages of 33, 16 times
        stages = [copy.deepcopy(protos[j % 4]) for j in range(64)]
        big = LIMIT_ALPHA if n_stages != 1 else "21.47483648"
        thr = LIMIT_THR if n_stages != 2 else "10995.11627776"
        stages[40]["alpha"][0:2] = [-float(big), float(big)]
        stages[40]["threshold"] = -float(thr)
        return _model(stages)
    if kind == "near_face":
        c = cascade_from_blob(load_cascade_blob())
        st = c["stage_classifier"][8]
        st["threshold"] = _dec(int(round(st["threshold"] * 1e8)) + 1, 8)
        return c
    raise ValueError(kind)


def cascade_corpus():
    """name -> (kind, seed, kwargs) of the synthetic corpus the table-driven cascade tests run (the JSON golden
    tests/golden/reference_js_cascades.json embeds each cascade, so its tests do not depend on this generator)."""
    corpus = {"ties": ("ties", 0, {}), "fp": ("fp", 0, {}), "shapes": ("shapes", 0, {}), "near_face": ("near_face", 0, {})}
    for n in (1, 2, 3, 7, 8, 9):
        corpus[f"short{n}"] = ("short", n, dict(n_stages=n))
        corpus[f"short{n}_fp"] = ("short", 100 if n == 1 else n, dict(n_stages=n, fp=True))   # (seed 1 draws no window)
    corpus["limits"] = ("limits", 0, {})
    corpus["limits_alpha"] = ("limits", 0, dict(n_stages=1))
    corpus["limits_thr"] = ("limits", 0, dict(n_stages=2))
    return corpus


def cascade_from_blob(blob):
    """The src/cascade.js form of an HTC1 blob (unused slots read back as z = -1, x = y = 0, as the packer writes them)."""
    c = parse_blob(blob)
    stages = []
    for count, first, thr in c["stages"]:
        feats, alphas = [], []
        for f in c["features"][first: first + count]:
            d = {"size": f["size"]}
            for side in "pn":
                pts = f[side][: f["size"]]
                d[side + "z"], d[side + "x"], d[side + "y"] = ([p[i] for p in pts] for i in range(3))
            feats.append(d)
            alphas += [f["a_fail"], f["a_pass"]]
        stages.append({"count": count, "threshold": thr, "feature": feats, "alpha": alphas})
    return _model(stages)
