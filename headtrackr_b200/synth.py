"""Deterministic synthetic RGBA frames for tests and bench (integer-only, so every machine agrees).

The reference ships no sample images (SURVEY.md §4).  Noise alone yields zero detections, which
would make parity vacuous, so frames carry "faces" synthesised from the cascade itself
(SURVEY.md Appendix A1): a 24x24 template whose pixels are the +-alpha votes of every feature
point of `headtrackr.cascade` (/root/reference/src/cascade.js:19), resized and pasted with a
skin-like tint on a blurred-noise background.

frame(i) is a pure function of (seed_base + i, W, H): PCG64 integers + integer box blurs +
the canvas-shim bilinear resize (same definition as oracle/ht_oracle.h).
"""
import struct
from functools import lru_cache
from pathlib import Path

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
