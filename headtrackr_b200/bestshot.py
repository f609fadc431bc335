"""Host mirror of a tracker stream's best shot (DESIGN.md 2, "Best shots"; ht_tracker_set_best_shot): per track, the
crop tick whose candidate - the RGBA8 face crop of the best shot's size and scale - is sharpest.

The device scores every crop tick's candidate and steps the state during the tick (Context.tracker_set_best_shot,
the "bestShot" key of TrackerSet) on an ht_best_shot_state in device memory; score() and step() replay that from the
candidates and the tick's records.  The score is integer arithmetic on the detector's gray, so the three agree exactly.

A state is a dict with the fields of ht_best_shot_state, as state_from_bytes decodes it; new_state() is the state a
best shot starts with.
"""
import numpy as np

from . import _lib
from .framing import crop_tick

BEGAN, IMPROVED, ENDED = _lib.HT_BEST_BEGAN, _lib.HT_BEST_IMPROVED, _lib.HT_BEST_ENDED
_FIELDS = [f for f, _ in _lib.BestShotState._fields_]


def gray(rgba):
    """the detector's gray of (..., 4) uint8 pixels, ccv.grayscale: R 0.3 + G 0.59 + B 0.11 in fp64, left to right,
    stored round-half-even"""
    p = np.asarray(rgba).astype(np.float64)
    v = (p[..., 0] * 0.3 + p[..., 1] * 0.59) + p[..., 2] * 0.11
    return np.minimum(np.rint(v), 255.0).astype(np.int64)


def score(rgba):
    """the best-shot score of an (S_h, S_w, 4) uint8 image (S_w, S_h >= 3): sum of L^2, L = 4 g(i,j) - g(i-1,j) -
    g(i+1,j) - g(i,j-1) - g(i,j+1), over the pixels 1 <= i <= S_w-2, 1 <= j <= S_h-2 whose alpha and whose four
    neighbours' alphas are all 255 -> int"""
    a = np.asarray(rgba)
    if a.ndim != 3 or a.shape[2] != 4 or a.shape[0] < 3 or a.shape[1] < 3:
        raise ValueError("a best-shot image is (S_h, S_w, 4) with S_w, S_h >= 3")
    g = gray(a)
    ok = a[..., 3] == 255
    c = g[1:-1, 1:-1]
    L = 4 * c - g[1:-1, :-2] - g[1:-1, 2:] - g[:-2, 1:-1] - g[2:, 1:-1]
    keep = ok[1:-1, 1:-1] & ok[1:-1, :-2] & ok[1:-1, 2:] & ok[:-2, 1:-1] & ok[2:, 1:-1]
    return int(np.sum(np.where(keep, L * L, 0), dtype=np.uint64))


def new_state():
    """the state a best shot starts with (and after it is set again): no track begun"""
    return {f: (0.0 if f in ("x", "y", "width", "height", "angle", "now_ms") else 0) for f in _FIELDS}


def end(state):
    """ends an open track (flags ENDED), as ht_tracker_import does; otherwise changes nothing"""
    if state["ended"] != state["track"]:
        state["ended"] = state["track"]
        state["flags"] = ENDED


def step(state, record, score, now_ms, canvas_w, canvas_h, two=True):
    """one tick of a stream's best shot (two: it has two images), in place: `record` a tracker record dict (detection
    "CS" / 2, x, y, width, height, angle), `score` its candidate's score (read only on a crop tick), now_ms its clock
    and canvas_w x canvas_h its canvas -> whether the tick set a new best (the candidate goes to image
    state["buffer"])"""
    state["flags"] = 0
    if not crop_tick(record):
        end(state)
        return False
    if state["ended"] == state["track"]:
        state["track"] = (state["track"] + 1) & 0xFFFFFFFF
        state["ticks"] = 0
        state["buffer"] = (state["track"] - 1) & 1 if two else 0
        state["flags"] = BEGAN
    state["score"] = int(score)
    best = state["ticks"] == 0 or int(score) > state["best_score"]
    if best:
        state["best_score"] = int(score)
        for k in ("x", "y", "width", "height", "angle"):
            state[k] = float(record[k])
        state.update(now_ms=float(now_ms), canvas_w=int(canvas_w), canvas_h=int(canvas_h), best_tick=state["ticks"])
        state["flags"] |= IMPROVED
    state["ticks"] += 1
    return best


def state_from_bytes(b):
    """an ht_best_shot_state (BEST_SHOT_STATE_BYTES bytes: numpy, bytes, or a torch tensor, copied to the host) ->
    state dict"""
    if hasattr(b, "detach"):
        b = b.detach().cpu().numpy()
    raw = bytes(memoryview(b).cast("B")) if not isinstance(b, (bytes, bytearray)) else bytes(b)
    if len(raw) != _lib.BEST_SHOT_STATE_BYTES:
        raise ValueError(f"an ht_best_shot_state is {_lib.BEST_SHOT_STATE_BYTES} bytes")
    s = _lib.BestShotState.from_buffer_copy(raw)
    return {f: getattr(s, f) for f in _FIELDS}


def state_to_bytes(state):
    """a state dict -> its ht_best_shot_state bytes"""
    return bytes(_lib.BestShotState(**state))
