"""headtrackr_b200 — H100-native (sm_90a) replacement for headtrackr's detect+track pixel kernels.

Host-side mirror of the reference's L1 interface (SURVEY.md §1):
    headtrackr_b200.ccv.grayscale / ccv.detect_objects      <- /root/reference/src/ccv.js
    headtrackr_b200.cascade                                  <- /root/reference/src/cascade.js
    headtrackr_b200.camshift.Tracker / Rectangle / TrackObj  <- /root/reference/src/camshift.js
    headtrackr_b200.getWhitebalance                          <- /root/reference/src/whitebalance.js
    headtrackr_b200.facetrackr.Tracker                       <- /root/reference/src/facetrackr.js (host state machine)
    headtrackr_b200.smoother.Smoother, headposition.Tracker  <- src/smoother.js, src/headposition.js (host scalars)
All pixel work runs in libheadtrackr_b200.so (CUDA, C ABI in include/headtrackr_b200.h).
"""
from . import _lib  # noqa: F401
from . import camshift, ccv, facetrackr, headposition, main, smoother  # noqa: F401
from .canvas import Canvas, as_pixels  # noqa: F401
from .context import Context  # noqa: F401
from .synth import load_cascade_blob  # noqa: F401


def cascade():
    """headtrackr.cascade (src/cascade.js:19) as the packed "HTC1" blob the C ABI consumes."""
    return load_cascade_blob()


def getWhitebalance(canvas, context=None):
    """headtrackr.getWhitebalance(canvas) — src/whitebalance.js:5-29 (average gray of the frame)."""
    from .runtime import default_context
    px = as_pixels(canvas)
    ctx = context or default_context(px.shape[1], px.shape[0])
    return float(ctx.whitebalance(px)[0])


__all__ = ["Context", "Canvas", "load_cascade_blob", "cascade", "getWhitebalance", "ccv", "camshift", "facetrackr", "smoother", "headposition"]
