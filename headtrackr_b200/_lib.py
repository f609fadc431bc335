"""ctypes binding of libheadtrackr_b200.so (C ABI: include/headtrackr_b200.h).

There is no CPU fallback: if the shared library is missing it is built with nvcc (sm_90a); if that
is impossible the import fails loudly.  Nothing here imports the oracle.
"""
import ctypes as C
import os
import shutil
import subprocess
from pathlib import Path

_PKG = Path(__file__).resolve().parent
# HT_LIB selects another build of the same library (A/B variants of compile-time knobs, tools/build_variants.sh)
SO_PATH = Path(os.environ["HT_LIB"]).resolve() if os.environ.get("HT_LIB") else _PKG / "libheadtrackr_b200.so"
CSRC = _PKG / "csrc"

HT_OK, HT_WARN_OVERFLOW = 0, 1
HT_ERR_ARG, HT_ERR_CUDA, HT_ERR_SIZE, HT_ERR_CASCADE, HT_ERR_STATE = -1, -2, -3, -4, -5


class HtError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"headtrackr_b200 error {code}: {msg}")
        self.code = code


class Rect(C.Structure):
    _fields_ = [("x", C.c_double), ("y", C.c_double), ("width", C.c_double), ("height", C.c_double),
                ("confidence", C.c_double), ("neighbors", C.c_int32), ("pad_", C.c_int32)]


class TrackObj(C.Structure):
    _fields_ = [("x", C.c_int32), ("y", C.c_int32), ("width", C.c_int32), ("height", C.c_int32),
                ("angle", C.c_double)]


class Window(C.Structure):
    _fields_ = [("x", C.c_int32), ("y", C.c_int32), ("width", C.c_int32), ("height", C.c_int32)]


class StreamEvent(C.Structure):
    _fields_ = [("detection", C.c_int32), ("status", C.c_int32), ("x", C.c_double), ("y", C.c_double),
                ("width", C.c_double), ("height", C.c_double), ("angle", C.c_double), ("confidence", C.c_double)]


class HeadParams(C.Structure):
    _fields_ = [("smoothing", C.c_int32), ("head_position", C.c_int32), ("edgecorrection", C.c_int32), ("pad_", C.c_int32),
                ("alpha", C.c_double), ("fov_deg", C.c_double), ("camera_offset", C.c_double),
                ("distance_to_screen", C.c_double)]


class HeadEvent(C.Structure):
    _fields_ = [("valid", C.c_int32), ("status", C.c_int32), ("x", C.c_double), ("y", C.c_double), ("z", C.c_double),
                ("fx", C.c_double), ("fy", C.c_double), ("fwidth", C.c_double), ("fheight", C.c_double)]


class TrackerParams(C.Structure):
    _fields_ = [("retry_detection", C.c_int32), ("calc_angles", C.c_int32), ("pad_", C.c_int32 * 2), ("head", HeadParams)]


class TrackerEvent(C.Structure):
    _fields_ = [("detection", C.c_int32), ("status", C.c_int32), ("x", C.c_double), ("y", C.c_double),
                ("width", C.c_double), ("height", C.c_double), ("angle", C.c_double), ("confidence", C.c_double),
                ("wb", C.c_double), ("running", C.c_int32), ("pad_", C.c_int32), ("fov", C.c_double), ("head", HeadEvent)]


class VideoFrame(C.Structure):
    """ht_video_frame: one stream's video frame for ht_tracker_feed (pitch 0 = 4 * width)"""
    _fields_ = [("rgba", C.c_void_p), ("stream", C.c_int32), ("width", C.c_int32), ("height", C.c_int32),
                ("pitch", C.c_int32), ("now_ms", C.c_double)]


class CanvasFrame(C.Structure):
    """ht_canvas_frame: one stream's video frame and its own working canvas for ht_tracker_feed_canvases"""
    _fields_ = [("video", VideoFrame), ("canvas_w", C.c_int32), ("canvas_h", C.c_int32), ("pad_", C.c_int32 * 2)]


# ht_yuv_image.format / .color
YUV_FORMATS = {"nv12": 0, "i420": 1, "nv21": 16, "i422": 17, "i444": 18, "yuyv": 19, "uyvy": 20, "p010": 21,
               "bgra": 32, "bgr24": 33, "rgb24": 34}
YUV_COLORS = {"bt601": 0, "bt709": 1, "bt601-full": 2, "bt709-full": 3, "bt2020": 8, "bt2020-full": 10}


class YuvImage(C.Structure):
    """ht_yuv_image: a video frame of one of YUV_FORMATS (the planes of each: include/headtrackr_b200.h; pitch 0 = the
    tight pitch)"""
    _fields_ = [("planes", C.c_void_p * 3), ("pitch", C.c_int32 * 3), ("width", C.c_int32), ("height", C.c_int32),
                ("format", C.c_int32), ("color", C.c_int32), ("pad_", C.c_int32)]


class YuvFrame(C.Structure):
    """ht_yuv_frame: one stream's YUV video frame, working canvas and clock for ht_tracker_feed_yuv"""
    _fields_ = [("video", YuvImage), ("stream", C.c_int32), ("canvas_w", C.c_int32), ("canvas_h", C.c_int32),
                ("pad_", C.c_int32), ("now_ms", C.c_double)]


assert C.sizeof(YuvImage) == 56 and C.sizeof(YuvFrame) == 80 and YuvFrame.now_ms.offset == 72

# ht_video_view.orientation: orientation & 3 = clockwise quarter turns, then HT_VIEW_MIRROR mirrors horizontally
HT_VIEW_ROTATE_90, HT_VIEW_ROTATE_180, HT_VIEW_ROTATE_270, HT_VIEW_MIRROR = 1, 2, 3, 4


class VideoView(C.Structure):
    """ht_video_view: an orientation (0..7) and a source rectangle of the oriented frame (all 0 = the whole frame)"""
    _fields_ = [("orientation", C.c_int32), ("sx", C.c_int32), ("sy", C.c_int32), ("sw", C.c_int32), ("sh", C.c_int32),
                ("reserved", C.c_int32 * 3)]


class DebugCanvas(C.Structure):
    """ht_debug_canvas: a stream's debug canvas for ht_tracker_set_debug (device memory; rgba NULL = none; pitch 0 =
    4 * width)"""
    _fields_ = [("rgba", C.c_void_p), ("width", C.c_int32), ("height", C.c_int32), ("pitch", C.c_int32),
                ("pad_", C.c_int32)]


class FaceCrop(C.Structure):
    """ht_face_crop: a stream's face crop for ht_tracker_set_face_crop (device memory; rgba NULL = none; pitch 0 =
    4 * width; scale in (0, 16])"""
    _fields_ = [("rgba", C.c_void_p), ("width", C.c_int32), ("height", C.c_int32), ("pitch", C.c_int32),
                ("pad_", C.c_int32), ("scale", C.c_double)]


assert C.sizeof(FaceCrop) == 32


class FaceCropYuv(C.Structure):
    """ht_face_crop_yuv: a stream's face crop as NV12 or I420 for ht_tracker_set_face_crop_yuv (device planes; planes[0]
    NULL = none; pitch 0 = tight; even sizes; color one of the BT.601 / BT.709 YUV_COLORS; scale in (0, 16])"""
    _fields_ = [("planes", C.c_void_p * 3), ("pitch", C.c_int32 * 3), ("width", C.c_int32), ("height", C.c_int32),
                ("format", C.c_int32), ("color", C.c_int32), ("pad_", C.c_int32), ("scale", C.c_double)]


assert C.sizeof(FaceCropYuv) == 64 and FaceCropYuv.scale.offset == 56


# ht_face_tensor.dtype / .layout / .channels
HT_TENSOR_U8, HT_TENSOR_F16, HT_TENSOR_BF16, HT_TENSOR_F32 = 0, 1, 2, 3
HT_TENSOR_CHW, HT_TENSOR_HWC = 0, 1
HT_TENSOR_RGB, HT_TENSOR_BGR, HT_TENSOR_GRAY = 0, 1, 2


class FaceTensor(C.Structure):
    """ht_face_tensor: a stream's face as a model's input for ht_tracker_set_face_tensor (device memory; data NULL =
    none; strides in elements; the element (k, j, i) at k plane_stride + j row_stride + i (CHW) or j row_stride + i C + k
    (HWC); value fmaf(c, mul[k], add[k]) rounded to the dtype; scale in (0, 16])"""
    _fields_ = [("data", C.c_void_p), ("row_stride", C.c_int64), ("plane_stride", C.c_int64), ("width", C.c_int32),
                ("height", C.c_int32), ("dtype", C.c_int32), ("layout", C.c_int32), ("channels", C.c_int32),
                ("pad_", C.c_int32), ("mul", C.c_float * 3), ("add", C.c_float * 3), ("scale", C.c_double)]


assert C.sizeof(FaceTensor) == 80 and FaceTensor.width.offset == 24 and FaceTensor.mul.offset == 48 and \
    FaceTensor.add.offset == 60 and FaceTensor.scale.offset == 72


class Camera(C.Structure):
    """ht_camera: a stream's head-coupled camera (HT_CAMERA_BYTES, in device memory; camera_from_bytes decodes it)"""
    _fields_ = [("position", C.c_double * 3), ("fov", C.c_double), ("view", C.c_double * 6), ("events", C.c_uint32),
                ("has_view_offset", C.c_int32), ("projection", C.c_float * 16), ("view_matrix", C.c_float * 16),
                ("pad_", C.c_uint32 * 2)]


class CameraControl(C.Structure):
    """ht_camera_control: one stream's realisticAbsoluteCameraControl for ht_tracker_set_camera (camera NULL = none)"""
    _fields_ = [("camera", C.c_void_p), ("scaling", C.c_double), ("fixed_position", C.c_double * 3),
                ("look_at", C.c_double * 3), ("screen_height", C.c_double), ("damping", C.c_double),
                ("fov", C.c_double), ("aspect", C.c_double), ("near", C.c_double), ("far", C.c_double)]


CAMERA_BYTES = 224
assert C.sizeof(Camera) == CAMERA_BYTES and C.sizeof(CameraControl) == 112

# ht_framing.outputs
HT_FRAMING_CROP, HT_FRAMING_TENSOR = 1, 2


class FramedBox(C.Structure):
    """ht_framed_box: a stream's framed box, the state of its framing (FRAMED_BOX_BYTES, in device memory;
    framing.box_from_bytes decodes it)"""
    _fields_ = [("cx", C.c_double), ("cy", C.c_double), ("width", C.c_double), ("height", C.c_double),
                ("canvas_w", C.c_int32), ("canvas_h", C.c_int32), ("updates", C.c_uint32), ("valid", C.c_int32)]


class Framing(C.Structure):
    """ht_framing: one stream's framing for ht_tracker_set_framing (box NULL = none; alpha in (0, 1]; dead_zone in
    [0, 0.5]; outputs a nonzero mask of HT_FRAMING_CROP | HT_FRAMING_TENSOR)"""
    _fields_ = [("box", C.c_void_p), ("alpha", C.c_double), ("dead_zone", C.c_double), ("outputs", C.c_int32),
                ("pad_", C.c_int32)]


FRAMED_BOX_BYTES = 48
assert C.sizeof(FramedBox) == FRAMED_BOX_BYTES and FramedBox.canvas_w.offset == 32 and FramedBox.valid.offset == 44 \
    and C.sizeof(Framing) == 32 and Framing.outputs.offset == 24

# ht_face_redact.mode
HT_REDACT_OFF, HT_REDACT_MOSAIC, HT_REDACT_FILL = 0, 1, 2


class FaceRedact(C.Structure):
    """ht_face_redact: one stream's face redaction for ht_tracker_set_redact (mode HT_REDACT_OFF = none; block even in
    2..128; hold 0..65535 ticks; fill_rgb for RGBA8 and packed RGB video, fill_yuv for YUV video; scale in (0, 16])"""
    _fields_ = [("mode", C.c_int32), ("block", C.c_int32), ("hold", C.c_int32), ("fill_rgb", C.c_uint8 * 3),
                ("pad0", C.c_uint8), ("fill_yuv", C.c_uint8 * 3), ("pad1", C.c_uint8), ("pad_", C.c_int32),
                ("scale", C.c_double)]


assert C.sizeof(FaceRedact) == 32 and FaceRedact.fill_rgb.offset == 12 and FaceRedact.fill_yuv.offset == 16 \
    and FaceRedact.pad_.offset == 20 and FaceRedact.scale.offset == 24

# ht_best_shot_state.flags
HT_BEST_BEGAN, HT_BEST_IMPROVED, HT_BEST_ENDED = 1, 2, 4


class BestShotState(C.Structure):
    """ht_best_shot_state: a stream's best-shot state (BEST_SHOT_STATE_BYTES, in device memory; bestshot.state_from_bytes
    decodes it)"""
    _fields_ = [("best_score", C.c_uint64), ("score", C.c_uint64), ("x", C.c_double), ("y", C.c_double),
                ("width", C.c_double), ("height", C.c_double), ("angle", C.c_double), ("now_ms", C.c_double),
                ("canvas_w", C.c_int32), ("canvas_h", C.c_int32), ("track", C.c_uint32), ("ended", C.c_uint32),
                ("ticks", C.c_uint32), ("best_tick", C.c_uint32), ("buffer", C.c_int32), ("flags", C.c_uint32)]


class BestShot(C.Structure):
    """ht_best_shot: one stream's best shot for ht_tracker_set_best_shot (device memory; rgba[0] NULL = none, rgba[1]
    NULL = one image; 3..2048 pixels a side; pitch 0 = 4 * width; scale in (0, 16])"""
    _fields_ = [("rgba", C.c_void_p * 2), ("state", C.c_void_p), ("width", C.c_int32), ("height", C.c_int32),
                ("pitch", C.c_int32), ("pad_", C.c_int32), ("scale", C.c_double)]


BEST_SHOT_STATE_BYTES = 96
assert C.sizeof(BestShotState) == BEST_SHOT_STATE_BYTES and BestShotState.now_ms.offset == 56 \
    and BestShotState.track.offset == 72 and BestShotState.flags.offset == 92 and C.sizeof(BestShot) == 48 \
    and BestShot.state.offset == 16 and BestShot.scale.offset == 40

# ht_tracker_export / ht_tracker_import: bytes of one tracker record (HT_TRACKER_RECORD_BYTES)
TRACKER_RECORD_BYTES = 16864

# headtrackrStatus names of ht_tracker_event.status, bit 0 first (= the order src/main.js dispatches them in)
TRACKER_STATUS = ("whitebalance", "detecting", "hints", "redetecting", "lost", "stopped", "found")


class Config(C.Structure):
    _fields_ = [("device", C.c_int32), ("max_width", C.c_int32), ("max_height", C.c_int32),
                ("max_frames", C.c_int32), ("max_raw_per_frame", C.c_int32), ("max_rects_per_frame", C.c_int32),
                ("cuda_stream", C.c_void_p)]


def sources_newer_than_so():
    if not SO_PATH.exists():
        return True
    t = SO_PATH.stat().st_mtime
    srcs = list(CSRC.glob("*.cu")) + list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.inc")) + \
        [_PKG.parent / "include" / "headtrackr_b200.h"]
    return any(s.stat().st_mtime > t for s in srcs)


def nvcc():
    """The CUDA compiler: $CUDA_HOME/bin/nvcc, else nvcc on PATH, else the toolkit's default install prefix."""
    home = os.environ.get("CUDA_HOME") or os.environ.get("CUDA_PATH")
    if home and (Path(home) / "bin" / "nvcc").exists():
        return str(Path(home) / "bin" / "nvcc")
    return shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


def build(force=False):
    """Compile the sm_90a shared library in-tree (nvcc cross-compiles without a GPU)."""
    if force or sources_newer_than_so():
        subprocess.check_call(["make", "-s", "-C", str(CSRC), f"NVCC={nvcc()}"] + (["-B"] if force else []))
    if not SO_PATH.exists():
        raise ImportError(f"{SO_PATH} was not produced by the build")
    return SO_PATH


_lib = None

EXPORTS = ["ht_version", "ht_create", "ht_destroy", "ht_last_error", "ht_sync", "ht_max_rects", "ht_detect",
           "ht_track_init", "ht_track_init_from_detect", "ht_track", "ht_detect_track", "ht_stream_reset", "ht_stream_step", "ht_stream_head_config", "ht_stream_step_head",
           "ht_tracker_config", "ht_tracker_reset", "ht_tracker_start", "ht_tracker_stop", "ht_tracker_step", "ht_tracker_feed", "ht_tracker_set_params", "ht_tracker_feed_canvases", "ht_tracker_set_debug", "ht_tracker_set_debug_strokes", "ht_tracker_set_face_crop", "ht_tracker_set_face_crop_yuv", "ht_tracker_set_face_tensor", "ht_face_crop_map", "ht_tracker_set_framing", "ht_face_crop_map_framed", "ht_tracker_set_redact", "ht_face_redact_rect", "ht_tracker_set_best_shot", "ht_best_shot_score", "ht_tracker_set_camera", "ht_tracker_export", "ht_tracker_import", "ht_tracker_feed_yuv", "ht_ingest", "ht_ingest_yuv",
           "ht_tracker_feed_views", "ht_tracker_feed_yuv_views", "ht_ingest_views", "ht_ingest_yuv_views", "ht_backprojection", "ht_whitebalance",
           "ht_plan_info", "ht_debug_plane", "ht_debug_raw", "ht_debug_model_hist", "ht_debug_track_stats", "ht_set_track_memo", "ht_set_pipeline", "ht_join", "ht_debug_set_exactness", "ht_debug_track_trace", "ht_debug_track_phases", "ht_launch_count",
           "ht_profile", "ht_profile_read"]

PROF_CLASSES = ["gray", "pyramid", "cascade", "group", "hist", "track_init", "track"]


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not SO_PATH.exists():
        try:
            build()
        except Exception as e:  # no silent fallback
            raise ImportError(f"libheadtrackr_b200.so is missing and could not be built: {e}") from e
    L = C.CDLL(str(SO_PATH))
    vp = C.c_void_p  # raw addresses: host or device pointers
    L.ht_version.restype = C.c_uint32
    L.ht_create.argtypes = [C.POINTER(vp), C.POINTER(Config), C.c_char_p, C.c_size_t]
    L.ht_destroy.argtypes = [vp]
    L.ht_destroy.restype = None
    L.ht_last_error.argtypes = [vp]
    L.ht_last_error.restype = C.c_char_p
    L.ht_sync.argtypes = [vp]
    L.ht_max_rects.argtypes = [vp]
    L.ht_detect.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp]
    L.ht_track_init.argtypes = [vp, vp, C.c_int, vp, C.c_int, C.c_int, vp, C.c_int]
    L.ht_track_init_from_detect.argtypes = [vp, vp, C.c_int, vp, C.c_int, C.c_int, vp, vp, C.c_int, vp]
    L.ht_track.argtypes = [vp, vp, C.c_int, vp, C.c_int, C.c_int, C.c_int, vp, vp]
    L.ht_detect_track.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                  vp, vp, vp, vp, vp]
    L.ht_stream_reset.argtypes = [vp, C.c_int, C.c_int]
    L.ht_stream_step.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp]
    L.ht_stream_head_config.argtypes = [vp, vp]
    L.ht_stream_step_head.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp]
    L.ht_tracker_config.argtypes = [vp, vp]
    for f in (L.ht_tracker_reset, L.ht_tracker_start, L.ht_tracker_stop):
        f.argtypes = [vp, C.c_int, C.c_int]
    L.ht_tracker_step.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.c_double, vp]
    L.ht_tracker_feed.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp]
    L.ht_tracker_set_params.argtypes = [vp, C.c_int, C.c_int, vp]
    L.ht_tracker_feed_canvases.argtypes = [vp, vp, C.c_int, C.c_int, vp]
    L.ht_tracker_set_debug.argtypes = [vp, C.c_int, C.c_int, vp]
    L.ht_tracker_set_debug_strokes.argtypes = [vp, C.c_int, C.c_int, vp]
    L.ht_tracker_set_face_crop.argtypes = [vp, C.c_int, C.c_int, vp]
    L.ht_tracker_set_face_crop_yuv.argtypes = [vp, C.c_int, C.c_int, vp]
    L.ht_tracker_set_face_tensor.argtypes = [vp, C.c_int, C.c_int, vp]
    L.ht_face_crop_map.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp]
    L.ht_tracker_set_framing.argtypes = [vp, C.c_int, C.c_int, vp]
    L.ht_face_crop_map_framed.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp]
    L.ht_tracker_set_redact.argtypes = [vp, C.c_int, C.c_int, vp]
    L.ht_face_redact_rect.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp]
    L.ht_tracker_set_best_shot.argtypes = [vp, C.c_int, C.c_int, vp]
    L.ht_best_shot_score.argtypes = [vp, C.c_int, C.c_int, C.c_int, vp]
    L.ht_tracker_set_camera.argtypes = [vp, C.c_int, C.c_int, vp]
    L.ht_tracker_export.argtypes = [vp, vp, C.c_int, vp]
    L.ht_tracker_import.argtypes = [vp, vp, C.c_int, vp]
    L.ht_ingest.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, vp, C.c_int, C.c_int]
    L.ht_tracker_feed_yuv.argtypes = [vp, vp, C.c_int, C.c_int, vp]
    L.ht_ingest_yuv.argtypes = [vp, vp, C.c_int, C.c_int, vp, C.c_int, C.c_int]
    L.ht_tracker_feed_views.argtypes = [vp, vp, vp, C.c_int, C.c_int, vp]
    L.ht_tracker_feed_yuv_views.argtypes = [vp, vp, vp, C.c_int, C.c_int, vp]
    L.ht_ingest_views.argtypes = [vp, vp, vp, C.c_int, C.c_int, vp, C.c_int, C.c_int]
    L.ht_ingest_yuv_views.argtypes = [vp, vp, vp, C.c_int, C.c_int, vp, C.c_int, C.c_int]
    L.ht_backprojection.argtypes = [vp, C.c_int, vp, C.c_int, C.c_int, vp]
    L.ht_whitebalance.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, vp]
    L.ht_plan_info.argtypes = [vp, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp, C.c_int]
    L.ht_debug_plane.argtypes = [vp, C.c_int, C.c_int, C.c_int, vp, C.c_int, vp, vp]
    L.ht_debug_raw.argtypes = [vp, C.c_int, vp, C.c_int, vp]
    L.ht_debug_model_hist.argtypes = [vp, C.c_int, vp]
    L.ht_debug_track_stats.argtypes = [vp, vp, C.c_int]
    L.ht_debug_track_trace.argtypes = [vp, vp, C.c_int]
    L.ht_debug_track_phases.argtypes = [vp, vp, C.c_int]
    L.ht_set_track_memo.argtypes = [vp, C.c_int]
    L.ht_set_pipeline.argtypes = [vp, C.c_int]
    L.ht_join.argtypes = [vp]
    L.ht_debug_set_exactness.argtypes = [vp, C.c_int]
    L.ht_launch_count.argtypes = [vp]
    L.ht_launch_count.restype = C.c_uint64
    L.ht_profile.argtypes = [vp, C.c_int]
    L.ht_profile_read.argtypes = [vp, vp, vp, C.c_int]
    _lib = L
    return L
