// js/addon.cc — Node N-API binding of libheadtrackr_b200.so (include/headtrackr_b200.h).
//
// UNTESTED SOURCE: this image (and the GPU box) has no node, no node_api.h and no node-gyp, so this file
// cannot be compiled here (SURVEY.md §0 C4).  It is the thin binding a maintainer adds; all logic lives
// below the C ABI, which IS tested (tests/test_gpu_*.py through ctypes).  Build: `node-gyp rebuild` with
// js/binding.gyp on a machine with Node >= 12 and the CUDA runtime.
//
// Exposed to JavaScript (1:1 with the C ABI):
//   create(cascadeBlob: Buffer, {device,maxWidth,maxHeight,maxFrames}) -> handle (External)
//   detect(handle, rgba: Uint8ClampedArray|Buffer, n, w, h, interval, minNeighbors) -> Array<Array<rect>>
//   trackInit(handle, slot, rgba, w, h, x, y, rw, rh, calcAngles)
//   track(handle, slot, rgba, w, h, nCalls) -> {x,y,width,height,angle, window:{x,y,width,height}}
//   whitebalance(handle, rgba, w, h) -> Number
//   backprojection(handle, slot, rgba, w, h) -> Uint8ClampedArray
//   streamStep(handle, rgba /* n frames, one per stream */, n, w, h, interval, minNeighbors, calcAngles)
//        -> Array<{detection:"VJ"|"CS", x,y,width,height,angle,confidence, found, lost}>   (ht_stream_step)
//   streamReset(handle, first, n)
//   streamHeadConfig(handle, {smoothing, fov, cameraOffset, headPosition} | null)     (ht_stream_head_config)
//   streamStepHead(handle, rgba, n, w, h, interval, minNeighbors, calcAngles)
//        -> {events: [...as streamStep...], heads: Array<{valid, found, x, y, z}>}    (ht_stream_step_head)
//   ingest(handle, rgba /* n video frames */, n, sw, sh, dw, dh) -> Uint8ClampedArray (n canvases)   (ht_ingest)
//   trackerConfig(handle, {retryDetection, calcAngles, smoothing, fov, cameraOffset, headPosition} | null)
//   trackerReset / trackerStart / trackerStop(handle, first, n)
//   trackerStep(handle, rgba /* n canvases */, n, w, h, nowMs) -> Array<{detection, status: [...], running, fov, ...}>
//   trackerSetParams(handle, first, [params, ...])   (ht_tracker_set_params: each stream its own Tracker parameters)
//   trackerSetDebug(handle, first, [canvas|null, ...])  (ht_tracker_set_debug: each stream's debug canvas, device memory)
//   trackerSetDebugStrokes(handle, first, [bool, ...])  (ht_tracker_set_debug_strokes: main.js's strokes on the device)
//   trackerSetFaceCrop(handle, first, [crop|null, ...])  (ht_tracker_set_face_crop: each stream's face crop, device
//        memory)
//   trackerSetFaceCropYuv(handle, first, [crop|null, ...])  (ht_tracker_set_face_crop_yuv: each stream's NV12 / I420
//        face crop, device planes)
//   trackerSetFaceTensor(handle, first, [tensor|null, ...])  (ht_tracker_set_face_tensor: each stream's normalised
//        face tensor for a model, device memory)
//   trackerSetCamera(handle, first, [control|null, ...])  (ht_tracker_set_camera: each stream's head-coupled camera,
//        realisticAbsoluteCameraControl on an ht_camera in device memory)
//   trackerSetFraming(handle, first, [framing|null, ...])  (ht_tracker_set_framing: each stream's steady face-cam box,
//        an ht_framed_box in device memory, that its crop and / or tensor is cut from)
//   trackerSetRedact(handle, first, [redaction|null, ...])  (ht_tracker_set_redact: each stream's tracked face hidden
//        in its own device video after each tick, a mosaic or a fill)
//   trackerSetBestShot(handle, first, [shot|null, ...])  (ht_tracker_set_best_shot: each stream's sharpest face of its
//        current or last track, in one or two device RGBA8 images, with its state in device memory)
//   trackerExport(handle, [stream, ...]) -> Buffer of records; trackerImport(handle, [stream, ...], records)
//        (ht_tracker_export / ht_tracker_import: a stream's whole Tracker as HT_TRACKER_RECORD_BYTES per stream)
//   trackerFeed(handle, [{stream, rgba, width, height, nowMs, canvasWidth?, canvasHeight?}], canvasWidth, canvasHeight)
//        -> Array<record> (ht_tracker_feed_canvases: only the listed streams tick, each from its own video frame, clock
//        and canvas)
//   trackerFeedYuv(handle, [{stream, nowMs, canvasWidth, canvasHeight, format, color, width, height, y, uv | u, v}])
//        -> Array<record> (ht_tracker_feed_yuv: NV12 / I420 host planes, tight pitches)
//   ingestYuv(handle, [{format, color, width, height, y, uv | u, v}], dw, dh) -> Uint8ClampedArray   (ht_ingest_yuv)
//   trackerFeedViews / trackerFeedYuvViews / ingestYuvViews: the same records with a "view" each, {rotate, mirror,
//     crop: [x, y, w, h]}; ingestViews(handle, [{width, height, rgba, view}], dw, dh)   (ht_*_views)
//   destroy(handle)
#include <node_api.h>

#include <cstdint>
#include <cstring>
#include <initializer_list>
#include <vector>

#include "../include/headtrackr_b200.h"

#define NAPI_OK(call)                                             \
  do {                                                            \
    if ((call) != napi_ok) {                                      \
      napi_throw_error(env, nullptr, "N-API call failed: " #call); \
      return nullptr;                                             \
    }                                                             \
  } while (0)

static napi_value Throw(napi_env env, ht_ctx *ctx, int rc) {
  const char *msg = ht_last_error(ctx);
  napi_throw_error(env, nullptr, (msg && *msg) ? msg : (rc == HT_ERR_CUDA ? "CUDA error" : "headtrackr_b200 error"));
  return nullptr;
}

static bool GetBytes(napi_env env, napi_value v, uint8_t **data, size_t *len) {
  bool is_buf = false, is_ta = false;
  napi_is_buffer(env, v, &is_buf);
  if (is_buf) return napi_get_buffer_info(env, v, reinterpret_cast<void **>(data), len) == napi_ok;
  napi_is_typedarray(env, v, &is_ta);
  if (!is_ta) return false;
  napi_typedarray_type t;
  napi_value ab;
  size_t off;
  return napi_get_typedarray_info(env, v, &t, len, reinterpret_cast<void **>(data), &ab, &off) == napi_ok;
}

static void Finalize(napi_env, void *p, void *) { ht_destroy(static_cast<ht_ctx *>(p)); }

static napi_value Create(napi_env env, napi_callback_info info) {
  size_t argc = 2;
  napi_value argv[2];
  NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
  uint8_t *blob;
  size_t blob_len;
  if (!GetBytes(env, argv[0], &blob, &blob_len)) return Throw(env, nullptr, HT_ERR_ARG);
  ht_config cfg;
  std::memset(&cfg, 0, sizeof(cfg));
  cfg.max_width = 1280; cfg.max_height = 720; cfg.max_frames = 16;
  auto geti = [&](const char *k, int32_t *dst) {
    napi_value v; bool has = false;
    if (argc > 1 && napi_has_named_property(env, argv[1], k, &has) == napi_ok && has &&
        napi_get_named_property(env, argv[1], k, &v) == napi_ok) napi_get_value_int32(env, v, dst);
  };
  geti("device", &cfg.device); geti("maxWidth", &cfg.max_width); geti("maxHeight", &cfg.max_height);
  geti("maxFrames", &cfg.max_frames);
  ht_ctx *ctx = nullptr;
  int rc = ht_create(&ctx, &cfg, blob, blob_len);
  if (rc != HT_OK) return Throw(env, nullptr, rc);
  napi_value ext;
  NAPI_OK(napi_create_external(env, ctx, Finalize, nullptr, &ext));
  return ext;
}

static ht_ctx *Ctx(napi_env env, napi_value v) {
  void *p = nullptr;
  napi_get_value_external(env, v, &p);
  return static_cast<ht_ctx *>(p);
}

static napi_value SetNum(napi_env env, napi_value obj, const char *k, double v) {
  napi_value n;
  napi_create_double(env, v, &n);
  napi_set_named_property(env, obj, k, n);
  return obj;
}

// detect(handle, rgba, n, w, h, interval, minNeighbors) -> [[{x,y,width,height,neighbors,confidence}]]
static napi_value Detect(napi_env env, napi_callback_info info) {
  size_t argc = 7;
  napi_value argv[7];
  NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
  ht_ctx *ctx = Ctx(env, argv[0]);
  uint8_t *rgba; size_t len;
  if (!GetBytes(env, argv[1], &rgba, &len)) return Throw(env, ctx, HT_ERR_ARG);
  int32_t n, w, h, interval, mn;
  napi_get_value_int32(env, argv[2], &n); napi_get_value_int32(env, argv[3], &w);
  napi_get_value_int32(env, argv[4], &h); napi_get_value_int32(env, argv[5], &interval);
  napi_get_value_int32(env, argv[6], &mn);
  if (len < (size_t)n * w * h * 4) return Throw(env, ctx, HT_ERR_ARG);
  const int K = ht_max_rects(ctx);
  std::vector<ht_rect> rects((size_t)n * K);
  std::vector<int32_t> counts(n);
  int rc = ht_detect(ctx, rgba, n, w, h, interval, mn, rects.data(), counts.data());
  if (rc < 0) return Throw(env, ctx, rc);
  napi_value out;
  NAPI_OK(napi_create_array_with_length(env, n, &out));
  for (int f = 0; f < n; ++f) {
    napi_value list;
    napi_create_array_with_length(env, counts[f], &list);
    for (int i = 0; i < counts[f]; ++i) {
      const ht_rect &r = rects[(size_t)f * K + i];
      napi_value o;
      napi_create_object(env, &o);
      SetNum(env, o, "x", r.x); SetNum(env, o, "y", r.y); SetNum(env, o, "width", r.width);
      SetNum(env, o, "height", r.height);
      SetNum(env, o, mn > 0 ? "neighbors" : "neighbor", r.neighbors);   // src/ccv.js:232 vs :301
      SetNum(env, o, "confidence", r.confidence);
      napi_set_element(env, list, i, o);
    }
    napi_set_element(env, out, f, list);
  }
  return out;
}

static napi_value TrackInit(napi_env env, napi_callback_info info) {
  size_t argc = 10;
  napi_value argv[10];
  NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
  ht_ctx *ctx = Ctx(env, argv[0]);
  int32_t slot, w, h, r[4], calc;
  uint8_t *rgba; size_t len;
  napi_get_value_int32(env, argv[1], &slot);
  if (!GetBytes(env, argv[2], &rgba, &len)) return Throw(env, ctx, HT_ERR_ARG);
  napi_get_value_int32(env, argv[3], &w); napi_get_value_int32(env, argv[4], &h);
  for (int i = 0; i < 4; ++i) napi_get_value_int32(env, argv[5 + i], &r[i]);
  napi_get_value_int32(env, argv[9], &calc);
  int rc = ht_track_init(ctx, &slot, 1, rgba, w, h, r, calc);
  if (rc < 0) return Throw(env, ctx, rc);
  return nullptr;
}

static napi_value Track(napi_env env, napi_callback_info info) {
  size_t argc = 6;
  napi_value argv[6];
  NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
  ht_ctx *ctx = Ctx(env, argv[0]);
  int32_t slot, w, h, n_calls;
  uint8_t *rgba; size_t len;
  napi_get_value_int32(env, argv[1], &slot);
  if (!GetBytes(env, argv[2], &rgba, &len)) return Throw(env, ctx, HT_ERR_ARG);
  napi_get_value_int32(env, argv[3], &w); napi_get_value_int32(env, argv[4], &h);
  napi_get_value_int32(env, argv[5], &n_calls);
  ht_trackobj o; ht_window win;
  int rc = ht_track(ctx, &slot, 1, rgba, w, h, n_calls, &o, &win);
  if (rc < 0) return Throw(env, ctx, rc);
  napi_value out, wo;
  napi_create_object(env, &out); napi_create_object(env, &wo);
  SetNum(env, out, "x", o.x); SetNum(env, out, "y", o.y); SetNum(env, out, "width", o.width);
  SetNum(env, out, "height", o.height); SetNum(env, out, "angle", o.angle);
  SetNum(env, wo, "x", win.x); SetNum(env, wo, "y", win.y); SetNum(env, wo, "width", win.width);
  SetNum(env, wo, "height", win.height);
  napi_set_named_property(env, out, "window", wo);
  return out;
}

// facetrackr's state machine for n streams in one call (src/facetrackr.js:67-126 + src/main.js:230-244 on the device)
static napi_value StreamStep(napi_env env, napi_callback_info info) {
  size_t argc = 8;
  napi_value argv[8];
  NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
  ht_ctx *ctx = Ctx(env, argv[0]);
  uint8_t *rgba; size_t len;
  int32_t n, w, h, interval, min_neighbors, calc;
  if (!GetBytes(env, argv[1], &rgba, &len)) return Throw(env, ctx, HT_ERR_ARG);
  napi_get_value_int32(env, argv[2], &n); napi_get_value_int32(env, argv[3], &w); napi_get_value_int32(env, argv[4], &h);
  napi_get_value_int32(env, argv[5], &interval); napi_get_value_int32(env, argv[6], &min_neighbors);
  napi_get_value_int32(env, argv[7], &calc);
  if (n <= 0 || len < (size_t)n * w * h * 4) return Throw(env, ctx, HT_ERR_ARG);
  std::vector<ht_stream_event> ev((size_t)n);
  int rc = ht_stream_step(ctx, rgba, n, w, h, interval, min_neighbors, calc, ev.data());
  if (rc < 0) return Throw(env, ctx, rc);
  napi_value out;
  napi_create_array_with_length(env, (size_t)n, &out);
  for (int k = 0; k < n; ++k) {
    napi_value o, s, b;
    napi_create_object(env, &o);
    napi_create_string_utf8(env, ev[k].detection == 2 ? "CS" : "VJ", 2, &s);
    napi_set_named_property(env, o, "detection", s);
    SetNum(env, o, "x", ev[k].x); SetNum(env, o, "y", ev[k].y); SetNum(env, o, "width", ev[k].width);
    SetNum(env, o, "height", ev[k].height); SetNum(env, o, "angle", ev[k].angle); SetNum(env, o, "confidence", ev[k].confidence);
    napi_get_boolean(env, (ev[k].status & 1) != 0, &b); napi_set_named_property(env, o, "found", b);
    napi_get_boolean(env, (ev[k].status & 2) != 0, &b); napi_set_named_property(env, o, "lost", b);
    napi_set_element(env, out, (uint32_t)k, o);
  }
  return out;
}

static bool GetBoolProp(napi_env env, napi_value obj, const char *k, bool dflt) {
  bool has = false; napi_value v; bool out = dflt;
  if (napi_has_named_property(env, obj, k, &has) == napi_ok && has && napi_get_named_property(env, obj, k, &v) == napi_ok) napi_get_value_bool(env, v, &out);
  return out;
}
static double GetNumProp(napi_env env, napi_value obj, const char *k, double dflt) {
  bool has = false; napi_value v; double out = dflt;
  if (napi_has_named_property(env, obj, k, &has) == napi_ok && has && napi_get_named_property(env, obj, k, &v) == napi_ok) napi_get_value_double(env, v, &out);
  return out;
}

// headtrackr.Tracker's {smoothing, fov, cameraOffset, headPosition} (src/main.js:35-56) for the GPU head epilogue
static napi_value StreamHeadConfig(napi_env env, napi_callback_info info) {
  size_t argc = 2;
  napi_value argv[2];
  NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
  ht_ctx *ctx = Ctx(env, argv[0]);
  napi_valuetype t;
  napi_typeof(env, argv[1], &t);
  int rc;
  if (t != napi_object) rc = ht_stream_head_config(ctx, nullptr);
  else {
    ht_head_params p;
    std::memset(&p, 0, sizeof(p));
    p.smoothing = GetBoolProp(env, argv[1], "smoothing", true);
    p.head_position = GetBoolProp(env, argv[1], "headPosition", true);
    p.edgecorrection = 1;
    p.alpha = 0.35;                                              // src/main.js:163
    p.fov_deg = GetNumProp(env, argv[1], "fov", 0.0);            // <= 0: estimate (src/main.js:283-288)
    p.camera_offset = GetNumProp(env, argv[1], "cameraOffset", 11.5);
    p.distance_to_screen = 60.0;
    rc = ht_stream_head_config(ctx, &p);
  }
  if (rc < 0) return Throw(env, ctx, rc);
  return nullptr;
}

static napi_value StreamStepHead(napi_env env, napi_callback_info info) {
  size_t argc = 8;
  napi_value argv[8];
  NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
  ht_ctx *ctx = Ctx(env, argv[0]);
  uint8_t *rgba; size_t len;
  int32_t n, w, h, interval, min_neighbors, calc;
  if (!GetBytes(env, argv[1], &rgba, &len)) return Throw(env, ctx, HT_ERR_ARG);
  napi_get_value_int32(env, argv[2], &n); napi_get_value_int32(env, argv[3], &w); napi_get_value_int32(env, argv[4], &h);
  napi_get_value_int32(env, argv[5], &interval); napi_get_value_int32(env, argv[6], &min_neighbors);
  napi_get_value_int32(env, argv[7], &calc);
  if (n <= 0 || len < (size_t)n * w * h * 4) return Throw(env, ctx, HT_ERR_ARG);
  std::vector<ht_stream_event> ev((size_t)n);
  std::vector<ht_head_event> he((size_t)n);
  int rc = ht_stream_step_head(ctx, rgba, n, w, h, interval, min_neighbors, calc, ev.data(), he.data());
  if (rc < 0) return Throw(env, ctx, rc);
  napi_value out, events, heads;
  napi_create_object(env, &out);
  napi_create_array_with_length(env, (size_t)n, &events);
  napi_create_array_with_length(env, (size_t)n, &heads);
  for (int k = 0; k < n; ++k) {
    napi_value o, s, b;
    napi_create_object(env, &o);
    napi_create_string_utf8(env, ev[k].detection == 2 ? "CS" : "VJ", 2, &s);
    napi_set_named_property(env, o, "detection", s);
    SetNum(env, o, "x", ev[k].x); SetNum(env, o, "y", ev[k].y); SetNum(env, o, "width", ev[k].width);
    SetNum(env, o, "height", ev[k].height); SetNum(env, o, "angle", ev[k].angle); SetNum(env, o, "confidence", ev[k].confidence);
    napi_get_boolean(env, (ev[k].status & 2) != 0, &b); napi_set_named_property(env, o, "lost", b);
    napi_set_element(env, events, (uint32_t)k, o);
    napi_value hobj;
    napi_create_object(env, &hobj);
    napi_get_boolean(env, he[k].valid != 0, &b); napi_set_named_property(env, hobj, "valid", b);
    napi_get_boolean(env, (he[k].status & 1) != 0, &b); napi_set_named_property(env, hobj, "found", b);
    SetNum(env, hobj, "x", he[k].x); SetNum(env, hobj, "y", he[k].y); SetNum(env, hobj, "z", he[k].z);
    napi_set_element(env, heads, (uint32_t)k, hobj);
  }
  napi_set_named_property(env, out, "events", events);
  napi_set_named_property(env, out, "heads", heads);
  return out;
}

// canvasContext.drawImage(video, 0, 0, dw, dh) for n frames (src/main.js:170)
static napi_value Ingest(napi_env env, napi_callback_info info) {
  size_t argc = 7;
  napi_value argv[7];
  NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
  ht_ctx *ctx = Ctx(env, argv[0]);
  uint8_t *rgba; size_t len;
  int32_t n, sw, sh, dw, dh;
  if (!GetBytes(env, argv[1], &rgba, &len)) return Throw(env, ctx, HT_ERR_ARG);
  napi_get_value_int32(env, argv[2], &n); napi_get_value_int32(env, argv[3], &sw); napi_get_value_int32(env, argv[4], &sh);
  napi_get_value_int32(env, argv[5], &dw); napi_get_value_int32(env, argv[6], &dh);
  if (n <= 0 || len < (size_t)n * sw * sh * 4) return Throw(env, ctx, HT_ERR_ARG);
  void *data; napi_value ab, ta;
  NAPI_OK(napi_create_arraybuffer(env, (size_t)n * dw * dh * 4, &data, &ab));
  int rc = ht_ingest(ctx, rgba, n, sw, sh, static_cast<uint8_t *>(data), dw, dh);
  if (rc < 0) return Throw(env, ctx, rc);
  NAPI_OK(napi_create_typedarray(env, napi_uint8_clamped_array, (size_t)n * dw * dh * 4, ab, 0, &ta));
  return ta;
}

static napi_value StreamReset(napi_env env, napi_callback_info info) {
  size_t argc = 3;
  napi_value argv[3];
  NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
  ht_ctx *ctx = Ctx(env, argv[0]);
  int32_t first, n;
  napi_get_value_int32(env, argv[1], &first); napi_get_value_int32(env, argv[2], &n);
  int rc = ht_stream_reset(ctx, first, n);
  if (rc < 0) return Throw(env, ctx, rc);
  return nullptr;
}

static napi_value Whitebalance(napi_env env, napi_callback_info info) {
  size_t argc = 4;
  napi_value argv[4];
  NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
  ht_ctx *ctx = Ctx(env, argv[0]);
  uint8_t *rgba; size_t len; int32_t w, h;
  if (!GetBytes(env, argv[1], &rgba, &len)) return Throw(env, ctx, HT_ERR_ARG);
  napi_get_value_int32(env, argv[2], &w); napi_get_value_int32(env, argv[3], &h);
  double v = 0;
  int rc = ht_whitebalance(ctx, rgba, 1, w, h, &v);
  if (rc < 0) return Throw(env, ctx, rc);
  napi_value out;
  napi_create_double(env, v, &out);
  return out;
}

static napi_value Backprojection(napi_env env, napi_callback_info info) {
  size_t argc = 5;
  napi_value argv[5];
  NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
  ht_ctx *ctx = Ctx(env, argv[0]);
  int32_t slot, w, h; uint8_t *rgba; size_t len;
  napi_get_value_int32(env, argv[1], &slot);
  if (!GetBytes(env, argv[2], &rgba, &len)) return Throw(env, ctx, HT_ERR_ARG);
  napi_get_value_int32(env, argv[3], &w); napi_get_value_int32(env, argv[4], &h);
  void *data; napi_value ab, ta;
  NAPI_OK(napi_create_arraybuffer(env, (size_t)w * h * 4, &data, &ab));
  int rc = ht_backprojection(ctx, slot, rgba, w, h, static_cast<uint8_t *>(data));
  if (rc < 0) return Throw(env, ctx, rc);
  NAPI_OK(napi_create_typedarray(env, napi_uint8_clamped_array, (size_t)w * h * 4, ab, 0, &ta));
  return ta;
}

// headtrackr.Tracker's {retryDetection, calcAngles, smoothing, fov, cameraOffset, headPosition} (src/main.js:35-56)
static ht_tracker_params TrackerParamsOf(napi_env env, napi_value o) {
  ht_tracker_params p;
  std::memset(&p, 0, sizeof(p));
  p.retry_detection = GetBoolProp(env, o, "retryDetection", true);
  p.calc_angles = GetBoolProp(env, o, "calcAngles", false);
  p.head.smoothing = GetBoolProp(env, o, "smoothing", true);
  p.head.head_position = GetBoolProp(env, o, "headPosition", true);
  p.head.edgecorrection = 1;
  p.head.alpha = 0.35;                                         // src/main.js:163
  p.head.fov_deg = GetNumProp(env, o, "fov", 0.0);             // <= 0: estimate (src/main.js:283-288)
  p.head.camera_offset = GetNumProp(env, o, "cameraOffset", 11.5);
  p.head.distance_to_screen = 60.0;
  return p;
}

// the same parameters, or null to switch the per-stream lifecycle off
static napi_value TrackerConfig(napi_env env, napi_callback_info info) {
  size_t argc = 2;
  napi_value argv[2];
  NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
  ht_ctx *ctx = Ctx(env, argv[0]);
  napi_valuetype t = napi_undefined;
  if (argc > 1) napi_typeof(env, argv[1], &t);
  int rc;
  if (t != napi_object) rc = ht_tracker_config(ctx, nullptr);
  else {
    const ht_tracker_params p = TrackerParamsOf(env, argv[1]);
    rc = ht_tracker_config(ctx, &p);
  }
  if (rc < 0) return Throw(env, ctx, rc);
  return nullptr;
}

// trackerSetParams(handle, first, [{retryDetection, calcAngles, ...}, ...]): stream first+i gets params[i]
static napi_value TrackerSetParams(napi_env env, napi_callback_info info) {
  size_t argc = 3;
  napi_value argv[3];
  NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
  ht_ctx *ctx = Ctx(env, argv[0]);
  int32_t first = 0;
  uint32_t n = 0;
  napi_get_value_int32(env, argv[1], &first);
  NAPI_OK(napi_get_array_length(env, argv[2], &n));
  std::vector<ht_tracker_params> ps(n);
  for (uint32_t i = 0; i < n; ++i) {
    napi_value r;
    NAPI_OK(napi_get_element(env, argv[2], i, &r));
    ps[i] = TrackerParamsOf(env, r);
  }
  int rc = ht_tracker_set_params(ctx, first, (int)n, ps.data());
  if (rc < 0) return Throw(env, ctx, rc);
  return nullptr;
}

// trackerSetDebug(handle, first, [{rgba: BigInt device address, width, height, pitch}, null, ...]): stream first+i
// gets canvases[i] (params.debug); null or undefined: none
static napi_value TrackerSetDebug(napi_env env, napi_callback_info info) {
  size_t argc = 3;
  napi_value argv[3];
  NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
  ht_ctx *ctx = Ctx(env, argv[0]);
  int32_t first = 0;
  uint32_t n = 0;
  napi_get_value_int32(env, argv[1], &first);
  NAPI_OK(napi_get_array_length(env, argv[2], &n));
  std::vector<ht_debug_canvas> cs(n, ht_debug_canvas{nullptr, 0, 0, 0, 0});
  for (uint32_t i = 0; i < n; ++i) {
    napi_value r, v;
    napi_valuetype t = napi_undefined;
    NAPI_OK(napi_get_element(env, argv[2], i, &r));
    napi_typeof(env, r, &t);
    if (t != napi_object) continue;
    uint64_t addr = 0;
    bool lossless = false;
    if (napi_get_named_property(env, r, "rgba", &v) == napi_ok) napi_get_value_bigint_uint64(env, v, &addr, &lossless);
    cs[i].rgba = reinterpret_cast<uint8_t *>(static_cast<uintptr_t>(addr));
    if (napi_get_named_property(env, r, "width", &v) == napi_ok) napi_get_value_int32(env, v, &cs[i].width);
    if (napi_get_named_property(env, r, "height", &v) == napi_ok) napi_get_value_int32(env, v, &cs[i].height);
    if (napi_get_named_property(env, r, "pitch", &v) == napi_ok) napi_get_value_int32(env, v, &cs[i].pitch);
  }
  int rc = ht_tracker_set_debug(ctx, first, (int)n, cs.data());
  if (rc < 0) return Throw(env, ctx, rc);
  return nullptr;
}

// trackerSetDebugStrokes(handle, first, [bool, ...]): stream first+i strokes main.js's face rectangles onto its debug
// canvas when flags[i] is truthy
static napi_value TrackerSetDebugStrokes(napi_env env, napi_callback_info info) {
  size_t argc = 3;
  napi_value argv[3];
  NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
  ht_ctx *ctx = Ctx(env, argv[0]);
  int32_t first = 0;
  uint32_t n = 0;
  napi_get_value_int32(env, argv[1], &first);
  NAPI_OK(napi_get_array_length(env, argv[2], &n));
  std::vector<int32_t> flags(n, 0);
  for (uint32_t i = 0; i < n; ++i) {
    napi_value r, b;
    bool on = false;
    NAPI_OK(napi_get_element(env, argv[2], i, &r));
    if (napi_coerce_to_bool(env, r, &b) == napi_ok) napi_get_value_bool(env, b, &on);
    flags[i] = on ? 1 : 0;
  }
  int rc = ht_tracker_set_debug_strokes(ctx, first, (int)n, flags.data());
  if (rc < 0) return Throw(env, ctx, rc);
  return nullptr;
}

// trackerSetFaceCrop(handle, first, [{rgba: BigInt device address, width, height, pitch, scale}, null, ...]): stream
// first+i gets crops[i] (scale defaults to 1); null or undefined: none
static napi_value TrackerSetFaceCrop(napi_env env, napi_callback_info info) {
  size_t argc = 3;
  napi_value argv[3];
  NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
  ht_ctx *ctx = Ctx(env, argv[0]);
  int32_t first = 0;
  uint32_t n = 0;
  napi_get_value_int32(env, argv[1], &first);
  NAPI_OK(napi_get_array_length(env, argv[2], &n));
  std::vector<ht_face_crop> cs(n, ht_face_crop{nullptr, 0, 0, 0, 0, 1.0});
  for (uint32_t i = 0; i < n; ++i) {
    napi_value r, v;
    napi_valuetype t = napi_undefined;
    NAPI_OK(napi_get_element(env, argv[2], i, &r));
    napi_typeof(env, r, &t);
    if (t != napi_object) continue;
    uint64_t addr = 0;
    bool lossless = false;
    if (napi_get_named_property(env, r, "rgba", &v) == napi_ok) napi_get_value_bigint_uint64(env, v, &addr, &lossless);
    cs[i].rgba = reinterpret_cast<uint8_t *>(static_cast<uintptr_t>(addr));
    if (napi_get_named_property(env, r, "width", &v) == napi_ok) napi_get_value_int32(env, v, &cs[i].width);
    if (napi_get_named_property(env, r, "height", &v) == napi_ok) napi_get_value_int32(env, v, &cs[i].height);
    if (napi_get_named_property(env, r, "pitch", &v) == napi_ok) napi_get_value_int32(env, v, &cs[i].pitch);
    napi_valuetype st = napi_undefined;
    if (napi_get_named_property(env, r, "scale", &v) == napi_ok && napi_typeof(env, v, &st) == napi_ok && st == napi_number)
      napi_get_value_double(env, v, &cs[i].scale);
  }
  int rc = ht_tracker_set_face_crop(ctx, first, (int)n, cs.data());
  if (rc < 0) return Throw(env, ctx, rc);
  return nullptr;
}

static double GetNumber(napi_env env, napi_value obj, const char *name, double dflt);

// trackerSetFaceCropYuv(handle, first, [{y, uv | u, v: BigInt device addresses, yPitch?, uvPitch? | uPitch?, vPitch?,
// width, height, format: "nv12" | "i420", color: "bt601" | "bt709" | "bt601-full" | "bt709-full", scale?}, null, ...]):
// stream first+i gets crops[i] (pitches default to tight, scale to 1); null or undefined: none
static napi_value TrackerSetFaceCropYuv(napi_env env, napi_callback_info info) {
  size_t argc = 3;
  napi_value argv[3];
  NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
  ht_ctx *ctx = Ctx(env, argv[0]);
  int32_t first = 0;
  uint32_t n = 0;
  napi_get_value_int32(env, argv[1], &first);
  NAPI_OK(napi_get_array_length(env, argv[2], &n));
  std::vector<ht_face_crop_yuv> cs(n, ht_face_crop_yuv{{nullptr, nullptr, nullptr}, {0, 0, 0}, 0, 0, HT_YUV_NV12, HT_YUV_BT601, 0, 1.0});
  for (uint32_t i = 0; i < n; ++i) {
    napi_value r, v;
    napi_valuetype t = napi_undefined;
    NAPI_OK(napi_get_element(env, argv[2], i, &r));
    napi_typeof(env, r, &t);
    if (t != napi_object) continue;
    char s[16] = {0};
    size_t sl = 0;
    if (napi_get_named_property(env, r, "format", &v) == napi_ok) napi_get_value_string_utf8(env, v, s, sizeof s, &sl);
    const bool nv12 = strcmp(s, "i420") != 0;
    cs[i].format = strcmp(s, "nv12") == 0 ? HT_YUV_NV12 : nv12 ? -1 : HT_YUV_I420;
    static const struct { const char *name; int32_t code; } colors[] = {
        {"bt601", HT_YUV_BT601}, {"bt709", HT_YUV_BT709}, {"bt601-full", HT_YUV_FULL_RANGE},
        {"bt709-full", HT_YUV_BT709 | HT_YUV_FULL_RANGE}};
    sl = 0;
    s[0] = 0;
    if (napi_get_named_property(env, r, "color", &v) == napi_ok) napi_get_value_string_utf8(env, v, s, sizeof s, &sl);
    cs[i].color = sl == 0 ? HT_YUV_BT601 : -1;
    for (const auto &c : colors)
      if (strcmp(s, c.name) == 0) cs[i].color = c.code;
    const char *planes[3] = {"y", nv12 ? "uv" : "u", "v"}, *pitches[3] = {"yPitch", nv12 ? "uvPitch" : "uPitch", "vPitch"};
    for (int p = 0; p < (nv12 ? 2 : 3); ++p) {
      uint64_t addr = 0;
      bool lossless = false;
      if (napi_get_named_property(env, r, planes[p], &v) == napi_ok) napi_get_value_bigint_uint64(env, v, &addr, &lossless);
      cs[i].planes[p] = reinterpret_cast<uint8_t *>(static_cast<uintptr_t>(addr));
      cs[i].pitch[p] = (int32_t)GetNumber(env, r, pitches[p], 0.0);
    }
    if (napi_get_named_property(env, r, "width", &v) == napi_ok) napi_get_value_int32(env, v, &cs[i].width);
    if (napi_get_named_property(env, r, "height", &v) == napi_ok) napi_get_value_int32(env, v, &cs[i].height);
    cs[i].scale = GetNumber(env, r, "scale", 1.0);
  }
  int rc = ht_tracker_set_face_crop_yuv(ctx, first, (int)n, cs.data());
  if (rc < 0) return Throw(env, ctx, rc);
  return nullptr;
}

static double GetNumber(napi_env env, napi_value obj, const char *name, double dflt) {
  napi_value v;
  napi_valuetype t = napi_undefined;
  double d = dflt;
  if (napi_get_named_property(env, obj, name, &v) == napi_ok && napi_typeof(env, v, &t) == napi_ok && t == napi_number)
    napi_get_value_double(env, v, &d);
  return d;
}

static void GetVec3(napi_env env, napi_value obj, const char *name, double out[3]) {
  napi_value v, e;
  for (int i = 0; i < 3; ++i) out[i] = 0.0;
  if (napi_get_named_property(env, obj, name, &v) != napi_ok) return;
  for (uint32_t i = 0; i < 3; ++i)
    if (napi_get_element(env, v, i, &e) == napi_ok) napi_get_value_double(env, e, &out[i]);
}

// trackerSetFaceTensor(handle, first, [{data: BigInt device address, rowStride, planeStride?, width, height,
// dtype: "u8" | "f16" | "bf16" | "f32", layout: "chw" | "hwc", channels: "rgb" | "bgr" | "gray", mul: [3], add: [3],
// scale?}, null, ...]): stream first+i gets tensors[i] (strides in elements; mul defaults to 1, add to 0, scale to 1);
// null or undefined: none
static napi_value TrackerSetFaceTensor(napi_env env, napi_callback_info info) {
  size_t argc = 3;
  napi_value argv[3];
  NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
  ht_ctx *ctx = Ctx(env, argv[0]);
  int32_t first = 0;
  uint32_t n = 0;
  napi_get_value_int32(env, argv[1], &first);
  NAPI_OK(napi_get_array_length(env, argv[2], &n));
  std::vector<ht_face_tensor> ts(n, ht_face_tensor{});
  auto pick = [&](napi_value r, const char *name, std::initializer_list<const char *> names, int32_t dflt) {
    napi_value v;
    char s[16] = {0};
    size_t sl = 0;
    if (napi_get_named_property(env, r, name, &v) == napi_ok) napi_get_value_string_utf8(env, v, s, sizeof s, &sl);
    if (sl == 0) return dflt;
    int32_t code = 0;
    for (const char *nm : names) {
      if (strcmp(s, nm) == 0) return code;
      ++code;
    }
    return (int32_t)-1;                     // the library rejects it
  };
  for (uint32_t i = 0; i < n; ++i) {
    napi_value r, v;
    napi_valuetype t = napi_undefined;
    NAPI_OK(napi_get_element(env, argv[2], i, &r));
    napi_typeof(env, r, &t);
    if (t != napi_object) continue;
    ht_face_tensor &f = ts[i];
    uint64_t addr = 0;
    bool lossless = false;
    if (napi_get_named_property(env, r, "data", &v) == napi_ok) napi_get_value_bigint_uint64(env, v, &addr, &lossless);
    f.data = reinterpret_cast<void *>(static_cast<uintptr_t>(addr));
    f.row_stride = (int64_t)GetNumber(env, r, "rowStride", 0.0);
    f.plane_stride = (int64_t)GetNumber(env, r, "planeStride", 0.0);
    if (napi_get_named_property(env, r, "width", &v) == napi_ok) napi_get_value_int32(env, v, &f.width);
    if (napi_get_named_property(env, r, "height", &v) == napi_ok) napi_get_value_int32(env, v, &f.height);
    f.dtype = pick(r, "dtype", {"u8", "f16", "bf16", "f32"}, HT_TENSOR_F16);
    f.layout = pick(r, "layout", {"chw", "hwc"}, HT_TENSOR_CHW);
    f.channels = pick(r, "channels", {"rgb", "bgr", "gray"}, HT_TENSOR_RGB);
    double mul[3], add[3];
    GetVec3(env, r, "mul", mul);
    GetVec3(env, r, "add", add);
    napi_value mv;
    const bool has_mul = napi_get_named_property(env, r, "mul", &mv) == napi_ok && napi_typeof(env, mv, &t) == napi_ok &&
                         t == napi_object;
    for (int k = 0; k < 3; ++k) f.mul[k] = has_mul ? (float)mul[k] : 1.0f, f.add[k] = (float)add[k];
    f.scale = GetNumber(env, r, "scale", 1.0);
  }
  int rc = ht_tracker_set_face_tensor(ctx, first, (int)n, ts.data());
  if (rc < 0) return Throw(env, ctx, rc);
  return nullptr;
}

// trackerSetCamera(handle, first, [{camera: BigInt device address, scaling, fixedPosition: [x, y, z], lookAt: [x, y, z],
// screenHeight?, damping?, fov, aspect, near, far}, null, ...]): stream first+i gets controls[i]; null or undefined:
// none.  screenHeight and damping default to the reference's 20 and 1 (src/controllers.js:31-38).
static napi_value TrackerSetCamera(napi_env env, napi_callback_info info) {
  size_t argc = 3;
  napi_value argv[3];
  NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
  ht_ctx *ctx = Ctx(env, argv[0]);
  int32_t first = 0;
  uint32_t n = 0;
  napi_get_value_int32(env, argv[1], &first);
  NAPI_OK(napi_get_array_length(env, argv[2], &n));
  std::vector<ht_camera_control> cs(n);
  memset(cs.data(), 0, n * sizeof(ht_camera_control));
  for (uint32_t i = 0; i < n; ++i) {
    napi_value r, v;
    napi_valuetype t = napi_undefined;
    NAPI_OK(napi_get_element(env, argv[2], i, &r));
    napi_typeof(env, r, &t);
    if (t != napi_object) continue;
    uint64_t addr = 0;
    bool lossless = false;
    if (napi_get_named_property(env, r, "camera", &v) == napi_ok) napi_get_value_bigint_uint64(env, v, &addr, &lossless);
    ht_camera_control &c = cs[i];
    c.camera = reinterpret_cast<ht_camera *>(static_cast<uintptr_t>(addr));
    c.scaling = GetNumber(env, r, "scaling", 0.0);
    GetVec3(env, r, "fixedPosition", c.fixed_position);
    GetVec3(env, r, "lookAt", c.look_at);
    c.screen_height = GetNumber(env, r, "screenHeight", 20.0);
    c.damping = GetNumber(env, r, "damping", 1.0);
    c.fov = GetNumber(env, r, "fov", 0.0);
    c.aspect = GetNumber(env, r, "aspect", 0.0);
    c.near = GetNumber(env, r, "near", 0.0);
    c.far = GetNumber(env, r, "far", 0.0);
  }
  int rc = ht_tracker_set_camera(ctx, first, (int)n, cs.data());
  if (rc < 0) return Throw(env, ctx, rc);
  return nullptr;
}

// trackerSetFraming(handle, first, [{box: BigInt device address, alpha?, deadZone?, crop?, tensor?}, null, ...]): stream
// first+i gets framings[i]; null or undefined: none.  alpha and deadZone default to 0.25 and 0.1, crop to true and
// tensor to false, as in the Python wrapper.
static napi_value TrackerSetFraming(napi_env env, napi_callback_info info) {
  size_t argc = 3;
  napi_value argv[3];
  NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
  ht_ctx *ctx = Ctx(env, argv[0]);
  int32_t first = 0;
  uint32_t n = 0;
  napi_get_value_int32(env, argv[1], &first);
  NAPI_OK(napi_get_array_length(env, argv[2], &n));
  std::vector<ht_framing> fs(n);
  memset(fs.data(), 0, n * sizeof(ht_framing));
  for (uint32_t i = 0; i < n; ++i) {
    napi_value r, v;
    napi_valuetype t = napi_undefined;
    NAPI_OK(napi_get_element(env, argv[2], i, &r));
    napi_typeof(env, r, &t);
    if (t != napi_object) continue;
    uint64_t addr = 0;
    bool lossless = false;
    if (napi_get_named_property(env, r, "box", &v) == napi_ok) napi_get_value_bigint_uint64(env, v, &addr, &lossless);
    ht_framing &f = fs[i];
    f.box = reinterpret_cast<ht_framed_box *>(static_cast<uintptr_t>(addr));
    f.alpha = GetNumber(env, r, "alpha", 0.25);
    f.dead_zone = GetNumber(env, r, "deadZone", 0.1);
    bool crop = true, tensor = false;
    if (napi_get_named_property(env, r, "crop", &v) == napi_ok) napi_get_value_bool(env, v, &crop);
    if (napi_get_named_property(env, r, "tensor", &v) == napi_ok) napi_get_value_bool(env, v, &tensor);
    f.outputs = (crop ? HT_FRAMING_CROP : 0) | (tensor ? HT_FRAMING_TENSOR : 0);
  }
  int rc = ht_tracker_set_framing(ctx, first, (int)n, fs.data());
  if (rc < 0) return Throw(env, ctx, rc);
  return nullptr;
}

// trackerSetBestShot(handle, first, [{rgba: BigInt device address | [BigInt, BigInt], state: BigInt device address,
// width, height, pitch?, scale?}, null, ...]): stream first+i gets shots[i]; null or undefined: none.  pitch defaults
// to 4 * width and scale to 1, as in the Python wrapper.
static napi_value TrackerSetBestShot(napi_env env, napi_callback_info info) {
  size_t argc = 3;
  napi_value argv[3];
  NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
  ht_ctx *ctx = Ctx(env, argv[0]);
  int32_t first = 0;
  uint32_t n = 0;
  napi_get_value_int32(env, argv[1], &first);
  NAPI_OK(napi_get_array_length(env, argv[2], &n));
  std::vector<ht_best_shot> bs(n);
  memset(bs.data(), 0, n * sizeof(ht_best_shot));
  for (uint32_t i = 0; i < n; ++i) {
    napi_value r, v;
    napi_valuetype t = napi_undefined;
    NAPI_OK(napi_get_element(env, argv[2], i, &r));
    napi_typeof(env, r, &t);
    if (t != napi_object) continue;
    ht_best_shot &b = bs[i];
    bool lossless = false, pair = false;
    uint64_t addr[2] = {0, 0}, state = 0;
    if (napi_get_named_property(env, r, "rgba", &v) == napi_ok) {
      napi_is_array(env, v, &pair);
      if (pair) {
        for (uint32_t k = 0; k < 2; ++k) {
          napi_value e;
          if (napi_get_element(env, v, k, &e) == napi_ok) napi_get_value_bigint_uint64(env, e, &addr[k], &lossless);
        }
      } else {
        napi_get_value_bigint_uint64(env, v, &addr[0], &lossless);
      }
    }
    if (napi_get_named_property(env, r, "state", &v) == napi_ok) napi_get_value_bigint_uint64(env, v, &state, &lossless);
    for (int k = 0; k < 2; ++k) b.rgba[k] = reinterpret_cast<uint8_t *>(static_cast<uintptr_t>(addr[k]));
    b.state = reinterpret_cast<ht_best_shot_state *>(static_cast<uintptr_t>(state));
    b.width = (int32_t)GetNumber(env, r, "width", 0);
    b.height = (int32_t)GetNumber(env, r, "height", 0);
    b.pitch = (int32_t)GetNumber(env, r, "pitch", 0);
    b.scale = GetNumber(env, r, "scale", 1.0);
  }
  int rc = ht_tracker_set_best_shot(ctx, first, (int)n, bs.data());
  if (rc < 0) return Throw(env, ctx, rc);
  return nullptr;
}

// trackerSetRedact(handle, first, [{mode?: "mosaic" | "fill", block?, scale?, hold?, fillRgb?: [r, g, b],
// fillYuv?: [y, u, v]}, null, ...]): stream first+i gets redactions[i]; null or undefined: none.  The defaults are the
// Python wrapper's: mosaic, block 16, scale 1.25, hold 10, black.
static napi_value TrackerSetRedact(napi_env env, napi_callback_info info) {
  size_t argc = 3;
  napi_value argv[3];
  NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
  ht_ctx *ctx = Ctx(env, argv[0]);
  int32_t first = 0;
  uint32_t n = 0;
  napi_get_value_int32(env, argv[1], &first);
  NAPI_OK(napi_get_array_length(env, argv[2], &n));
  std::vector<ht_face_redact> rs(n);
  memset(rs.data(), 0, n * sizeof(ht_face_redact));
  for (uint32_t i = 0; i < n; ++i) {
    napi_value r, v;
    napi_valuetype t = napi_undefined;
    NAPI_OK(napi_get_element(env, argv[2], i, &r));
    napi_typeof(env, r, &t);
    if (t != napi_object) continue;
    ht_face_redact &d = rs[i];
    d.mode = HT_REDACT_MOSAIC;
    char mode[16] = "";
    size_t len = 0;
    if (napi_get_named_property(env, r, "mode", &v) == napi_ok &&
        napi_get_value_string_utf8(env, v, mode, sizeof(mode), &len) == napi_ok && strcmp(mode, "fill") == 0)
      d.mode = HT_REDACT_FILL;
    else if (len > 0 && strcmp(mode, "mosaic") != 0)
      d.mode = -1;                                   // refused by the library, naming the record
    d.block = (int32_t)GetNumber(env, r, "block", 16);
    d.hold = (int32_t)GetNumber(env, r, "hold", 10);
    d.scale = GetNumber(env, r, "scale", 1.25);
    const uint8_t yuv_black[3] = {16, 128, 128};
    for (int k = 0; k < 3; ++k) d.fill_yuv[k] = yuv_black[k];
    for (int c = 0; c < 2; ++c) {
      napi_value arr, e;
      bool is_array = false;
      if (napi_get_named_property(env, r, c ? "fillYuv" : "fillRgb", &arr) != napi_ok) continue;
      napi_is_array(env, arr, &is_array);
      for (uint32_t k = 0; is_array && k < 3; ++k) {
        int32_t x = 0;
        if (napi_get_element(env, arr, k, &e) == napi_ok && napi_get_value_int32(env, e, &x) == napi_ok)
          (c ? d.fill_yuv : d.fill_rgb)[k] = (uint8_t)x;
      }
    }
  }
  int rc = ht_tracker_set_redact(ctx, first, (int)n, rs.data());
  if (rc < 0) return Throw(env, ctx, rc);
  return nullptr;
}

// stream ids of an Array of numbers
static bool GetStreams(napi_env env, napi_value arr, std::vector<int32_t> *ids) {
  uint32_t n = 0;
  if (napi_get_array_length(env, arr, &n) != napi_ok) return false;
  ids->assign(n, -1);
  for (uint32_t i = 0; i < n; ++i) {
    napi_value v;
    if (napi_get_element(env, arr, i, &v) != napi_ok || napi_get_value_int32(env, v, &(*ids)[i]) != napi_ok) return false;
  }
  return true;
}

// trackerExport(handle, [stream, ...]) -> Buffer of streams.length tracker records (ht_tracker_export)
static napi_value TrackerExport(napi_env env, napi_callback_info info) {
  size_t argc = 2;
  napi_value argv[2];
  NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
  ht_ctx *ctx = Ctx(env, argv[0]);
  std::vector<int32_t> ids;
  if (!GetStreams(env, argv[1], &ids)) return Throw(env, ctx, HT_ERR_ARG);
  void *data = nullptr;
  napi_value buf;
  NAPI_OK(napi_create_buffer(env, ids.size() * HT_TRACKER_RECORD_BYTES, &data, &buf));
  int rc = ht_tracker_export(ctx, ids.data(), (int)ids.size(), data);
  if (rc < 0) return Throw(env, ctx, rc);
  return buf;
}

// trackerImport(handle, [stream, ...], records: Buffer | TypedArray of streams.length records) (ht_tracker_import)
static napi_value TrackerImport(napi_env env, napi_callback_info info) {
  size_t argc = 3;
  napi_value argv[3];
  NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
  ht_ctx *ctx = Ctx(env, argv[0]);
  std::vector<int32_t> ids;
  uint8_t *recs;
  size_t len;
  if (!GetStreams(env, argv[1], &ids) || !GetBytes(env, argv[2], &recs, &len) ||
      len != ids.size() * HT_TRACKER_RECORD_BYTES)
    return Throw(env, ctx, HT_ERR_ARG);
  int rc = ht_tracker_import(ctx, ids.data(), (int)ids.size(), recs);
  if (rc < 0) return Throw(env, ctx, rc);
  return nullptr;
}

// trackerReset / trackerStart / trackerStop(handle, first, n)
static napi_value TrackerRange(napi_env env, napi_callback_info info, int (*fn)(ht_ctx *, int, int)) {
  size_t argc = 3;
  napi_value argv[3];
  NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
  ht_ctx *ctx = Ctx(env, argv[0]);
  int32_t first, n;
  napi_get_value_int32(env, argv[1], &first); napi_get_value_int32(env, argv[2], &n);
  int rc = fn(ctx, first, n);
  if (rc < 0) return Throw(env, ctx, rc);
  return nullptr;
}
static napi_value TrackerReset(napi_env env, napi_callback_info info) { return TrackerRange(env, info, ht_tracker_reset); }
static napi_value TrackerStart(napi_env env, napi_callback_info info) { return TrackerRange(env, info, ht_tracker_start); }
static napi_value TrackerStop(napi_env env, napi_callback_info info) { return TrackerRange(env, info, ht_tracker_stop); }

static const char *kTrackerStatus[] = {"whitebalance", "detecting", "hints", "redetecting", "lost", "stopped", "found"};

// one ht_tracker_event -> {detection: ""|"VJ"|"CS"|"WB", x, y, width, height, angle, confidence, wb, running, fov,
// status: [headtrackrStatus messages in dispatch order], head: {valid, x, y, z}}
static napi_value TrackerEventObject(napi_env env, const ht_tracker_event &e) {
  static const char *kDet[] = {"", "VJ", "CS", "WB"};
  napi_value o, s, b, st, head;
  napi_create_object(env, &o);
  const char *det = (e.detection >= 0 && e.detection <= 3) ? kDet[e.detection] : "";
  napi_create_string_utf8(env, det, NAPI_AUTO_LENGTH, &s);
  napi_set_named_property(env, o, "detection", s);
  SetNum(env, o, "x", e.x); SetNum(env, o, "y", e.y); SetNum(env, o, "width", e.width); SetNum(env, o, "height", e.height);
  SetNum(env, o, "angle", e.angle); SetNum(env, o, "confidence", e.confidence); SetNum(env, o, "wb", e.wb);
  SetNum(env, o, "fov", e.fov);
  napi_get_boolean(env, e.running != 0, &b); napi_set_named_property(env, o, "running", b);
  napi_create_array(env, &st);
  uint32_t m = 0;
  for (int bit = 0; bit < 7; ++bit)
    if ((e.status >> bit) & 1) {
      napi_create_string_utf8(env, kTrackerStatus[bit], NAPI_AUTO_LENGTH, &s);
      napi_set_element(env, st, m++, s);
    }
  napi_set_named_property(env, o, "status", st);
  napi_create_object(env, &head);
  napi_get_boolean(env, e.head.valid != 0, &b); napi_set_named_property(env, head, "valid", b);
  SetNum(env, head, "x", e.head.x); SetNum(env, head, "y", e.head.y); SetNum(env, head, "z", e.head.z);
  napi_set_named_property(env, o, "head", head);
  return o;
}

// trackerStep(handle, rgba /* n canvases, one per stream */, n, w, h, nowMs) -> Array<record>   (ht_tracker_step)
static napi_value TrackerStep(napi_env env, napi_callback_info info) {
  size_t argc = 6;
  napi_value argv[6];
  NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
  ht_ctx *ctx = Ctx(env, argv[0]);
  uint8_t *rgba; size_t len;
  int32_t n, w, h;
  double now_ms;
  if (!GetBytes(env, argv[1], &rgba, &len)) return Throw(env, ctx, HT_ERR_ARG);
  napi_get_value_int32(env, argv[2], &n); napi_get_value_int32(env, argv[3], &w); napi_get_value_int32(env, argv[4], &h);
  napi_get_value_double(env, argv[5], &now_ms);
  if (n <= 0 || len < (size_t)n * w * h * 4) return Throw(env, ctx, HT_ERR_ARG);
  std::vector<ht_tracker_event> ev((size_t)n);
  int rc = ht_tracker_step(ctx, rgba, n, w, h, now_ms, ev.data());
  if (rc < 0) return Throw(env, ctx, rc);
  napi_value out;
  napi_create_array_with_length(env, (size_t)n, &out);
  for (int k = 0; k < n; ++k) napi_set_element(env, out, (uint32_t)k, TrackerEventObject(env, ev[k]));
  return out;
}

// trackerFeed(handle, [{stream, rgba, width, height, nowMs, canvasWidth?, canvasHeight?}], canvasWidth, canvasHeight)
// -> Array<record>, in record order (ht_tracker_feed_canvases with host frames: one tick of each listed stream on its
// own video, clock and canvas; a record without its own canvas size uses the call's)
// a record's optional "view": {rotate: 0 | 90 | 180 | 270, mirror: bool, crop: [x, y, w, h] of the oriented frame}
// -> an ht_video_view (absent: the identity view); false for a bad object
static bool ViewOf(napi_env env, napi_value r, ht_video_view *view) {
  std::memset(view, 0, sizeof(*view));
  bool has = false;
  napi_value v, c;
  if (napi_has_named_property(env, r, "view", &has) != napi_ok || !has) return true;
  if (napi_get_named_property(env, r, "view", &v) != napi_ok) return false;
  const int rotate = (int)GetNumProp(env, v, "rotate", 0);
  if (rotate != 0 && rotate != 90 && rotate != 180 && rotate != 270) return false;
  bool mirror = false;
  napi_value m;
  if (napi_has_named_property(env, v, "mirror", &has) == napi_ok && has && napi_get_named_property(env, v, "mirror", &m) == napi_ok)
    napi_get_value_bool(env, m, &mirror);
  view->orientation = rotate / 90 | (mirror ? HT_VIEW_MIRROR : 0);
  if (napi_has_named_property(env, v, "crop", &has) == napi_ok && has && napi_get_named_property(env, v, "crop", &c) == napi_ok) {
    napi_valuetype t;
    napi_typeof(env, c, &t);
    if (t != napi_null && t != napi_undefined) {
      uint32_t len = 0;
      if (napi_get_array_length(env, c, &len) != napi_ok || len != 4) return false;
      int32_t *dst[4] = {&view->sx, &view->sy, &view->sw, &view->sh};
      for (uint32_t i = 0; i < 4; ++i) {
        napi_value e;
        if (napi_get_element(env, c, i, &e) != napi_ok || napi_get_value_int32(env, e, dst[i]) != napi_ok) return false;
      }
    }
  }
  return true;
}

// trackerFeed(handle, records, cw, ch), and with views (each record's "view", ViewOf) ht_tracker_feed_views
static napi_value TrackerFeedAny(napi_env env, napi_callback_info info, bool with_views) {
  size_t argc = 4;
  napi_value argv[4];
  NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
  ht_ctx *ctx = Ctx(env, argv[0]);
  uint32_t n = 0;
  int32_t cw, ch;
  NAPI_OK(napi_get_array_length(env, argv[1], &n));
  napi_get_value_int32(env, argv[2], &cw); napi_get_value_int32(env, argv[3], &ch);
  if (n == 0) return Throw(env, ctx, HT_ERR_ARG);
  std::vector<ht_canvas_frame> frames(n);
  std::vector<ht_video_view> views(n);
  for (uint32_t b = 0; b < n; ++b) {
    napi_value r, v;
    NAPI_OK(napi_get_element(env, argv[1], b, &r));
    std::memset(&frames[b], 0, sizeof(frames[b]));
    if (!ViewOf(env, r, &views[b])) return Throw(env, ctx, HT_ERR_ARG);
    frames[b].canvas_w = (int32_t)GetNumProp(env, r, "canvasWidth", cw);
    frames[b].canvas_h = (int32_t)GetNumProp(env, r, "canvasHeight", ch);
    ht_video_frame &f = frames[b].video;
    f.stream = (int32_t)GetNumProp(env, r, "stream", -1);
    f.width = (int32_t)GetNumProp(env, r, "width", 0);
    f.height = (int32_t)GetNumProp(env, r, "height", 0);
    f.now_ms = GetNumProp(env, r, "nowMs", 0.0);
    uint8_t *rgba; size_t len;
    NAPI_OK(napi_get_named_property(env, r, "rgba", &v));
    if (!GetBytes(env, v, &rgba, &len) || len < (size_t)f.width * f.height * 4) return Throw(env, ctx, HT_ERR_ARG);
    f.rgba = rgba;
  }
  std::vector<ht_tracker_event> ev(n);
  int rc = with_views ? ht_tracker_feed_views(ctx, frames.data(), views.data(), (int)n, 0, ev.data())
                      : ht_tracker_feed_canvases(ctx, frames.data(), (int)n, 0, ev.data());
  if (rc < 0) return Throw(env, ctx, rc);
  napi_value out;
  napi_create_array_with_length(env, (size_t)n, &out);
  for (uint32_t b = 0; b < n; ++b) napi_set_element(env, out, b, TrackerEventObject(env, ev[b]));
  return out;
}

static napi_value TrackerFeed(napi_env env, napi_callback_info info) { return TrackerFeedAny(env, info, false); }
static napi_value TrackerFeedViews(napi_env env, napi_callback_info info) { return TrackerFeedAny(env, info, true); }

// a video frame object {format, color, width, height, planes}: format "nv12" (the default), "i420", "nv21", "i422",
// "i444", "yuyv", "uyvy", "p010", "bgra", "bgr24" or "rgb24"; color "bt601" (the default), "bt709", "bt2020", each
// optionally "-full"; planes under "y", "uv" (NV12, P010) / "vu" (NV21) / "u", "v", or "packed" for the packed formats
// (host Buffers / typed arrays, tight pitches) -> an ht_yuv_image; false for a bad object
static bool YuvImageOf(napi_env env, napi_value r, ht_yuv_image *img) {
  std::memset(img, 0, sizeof(*img));
  char s[16] = "";
  size_t sl = 0;
  napi_value v;
  bool has = false;
  img->width = (int32_t)GetNumProp(env, r, "width", 0);
  img->height = (int32_t)GetNumProp(env, r, "height", 0);
  if (img->width <= 0 || img->height <= 0) return false;
  if (napi_has_named_property(env, r, "format", &has) == napi_ok && has && napi_get_named_property(env, r, "format", &v) == napi_ok)
    napi_get_value_string_utf8(env, v, s, sizeof(s), &sl);
  static const struct { const char *name; int format; } formats[] = {
      {"nv12", HT_YUV_NV12}, {"i420", HT_YUV_I420}, {"nv21", HT_YUV_NV21}, {"i422", HT_YUV_I422}, {"i444", HT_YUV_I444},
      {"yuyv", HT_YUV_YUYV}, {"uyvy", HT_YUV_UYVY}, {"p010", HT_YUV_P010}, {"bgra", HT_YUV_BGRA},
      {"bgr24", HT_YUV_BGR24}, {"rgb24", HT_YUV_RGB24}};
  img->format = sl == 0 ? HT_YUV_NV12 : -1;
  for (const auto &f : formats)
    if (sl && std::strcmp(s, f.name) == 0) img->format = f.format;
  if (img->format < 0) return false;
  sl = 0;
  if (napi_has_named_property(env, r, "color", &has) == napi_ok && has && napi_get_named_property(env, r, "color", &v) == napi_ok)
    napi_get_value_string_utf8(env, v, s, sizeof(s), &sl);
  static const struct { const char *name; int color; } colors[] = {
      {"bt601", 0}, {"bt709", HT_YUV_BT709}, {"bt601-full", HT_YUV_FULL_RANGE},
      {"bt709-full", HT_YUV_BT709 | HT_YUV_FULL_RANGE}, {"bt2020", HT_YUV_BT2020},
      {"bt2020-full", HT_YUV_BT2020 | HT_YUV_FULL_RANGE}};
  img->color = sl == 0 ? HT_YUV_BT601 : -1;
  for (const auto &c : colors)
    if (sl && std::strcmp(s, c.name) == 0) img->color = c.color;
  const size_t w = (size_t)img->width, h = (size_t)img->height, cw = (w + 1) / 2, ch = (h + 1) / 2;
  const char *keys[3] = {"y", "uv", nullptr};
  size_t need[3] = {w * h, 2 * cw * ch, 0};
  switch (img->format) {
    case HT_YUV_NV21: keys[1] = "vu"; break;
    case HT_YUV_I420: keys[1] = "u", keys[2] = "v", need[1] = need[2] = cw * ch; break;
    case HT_YUV_I422: keys[1] = "u", keys[2] = "v", need[1] = need[2] = cw * h; break;
    case HT_YUV_I444: keys[1] = "u", keys[2] = "v", need[1] = need[2] = w * h; break;
    case HT_YUV_P010: need[0] = 2 * w * h, need[1] = 4 * cw * ch; break;
    case HT_YUV_YUYV: case HT_YUV_UYVY: keys[0] = "packed", keys[1] = nullptr, need[0] = 4 * cw * h; break;
    case HT_YUV_BGRA: keys[0] = "packed", keys[1] = nullptr, need[0] = 4 * w * h; break;
    case HT_YUV_BGR24: case HT_YUV_RGB24: keys[0] = "packed", keys[1] = nullptr, need[0] = 3 * w * h; break;
    default: break;
  }
  for (int p = 0; p < 3 && keys[p]; ++p) {
    uint8_t *data; size_t len;
    if (napi_get_named_property(env, r, keys[p], &v) != napi_ok || !GetBytes(env, v, &data, &len) || len < need[p]) return false;
    img->planes[p] = data;
  }
  return true;
}

// trackerFeedYuv(handle, [{stream, nowMs, canvasWidth, canvasHeight, ...a YUV frame object}]) -> Array<record>
// (ht_tracker_feed_yuv with host planes)
static napi_value TrackerFeedYuvAny(napi_env env, napi_callback_info info, bool with_views) {
  size_t argc = 2;
  napi_value argv[2];
  NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
  ht_ctx *ctx = Ctx(env, argv[0]);
  uint32_t n = 0;
  NAPI_OK(napi_get_array_length(env, argv[1], &n));
  if (n == 0) return Throw(env, ctx, HT_ERR_ARG);
  std::vector<ht_yuv_frame> frames(n);
  std::vector<ht_video_view> views(n);
  for (uint32_t b = 0; b < n; ++b) {
    napi_value r;
    NAPI_OK(napi_get_element(env, argv[1], b, &r));
    std::memset(&frames[b], 0, sizeof(frames[b]));
    if (!YuvImageOf(env, r, &frames[b].video) || !ViewOf(env, r, &views[b])) return Throw(env, ctx, HT_ERR_ARG);
    frames[b].stream = (int32_t)GetNumProp(env, r, "stream", -1);
    frames[b].canvas_w = (int32_t)GetNumProp(env, r, "canvasWidth", 0);
    frames[b].canvas_h = (int32_t)GetNumProp(env, r, "canvasHeight", 0);
    frames[b].now_ms = GetNumProp(env, r, "nowMs", 0.0);
  }
  std::vector<ht_tracker_event> ev(n);
  int rc = with_views ? ht_tracker_feed_yuv_views(ctx, frames.data(), views.data(), (int)n, 0, ev.data())
                      : ht_tracker_feed_yuv(ctx, frames.data(), (int)n, 0, ev.data());
  if (rc < 0) return Throw(env, ctx, rc);
  napi_value out;
  napi_create_array_with_length(env, (size_t)n, &out);
  for (uint32_t b = 0; b < n; ++b) napi_set_element(env, out, b, TrackerEventObject(env, ev[b]));
  return out;
}

static napi_value TrackerFeedYuv(napi_env env, napi_callback_info info) { return TrackerFeedYuvAny(env, info, false); }
static napi_value TrackerFeedYuvViews(napi_env env, napi_callback_info info) { return TrackerFeedYuvAny(env, info, true); }

// ingestYuv(handle, [YUV frame object, ...], dw, dh) -> Uint8ClampedArray (n canvases)   (ht_ingest_yuv); with views
// (each object's "view", ViewOf) ht_ingest_yuv_views
static napi_value IngestYuvAny(napi_env env, napi_callback_info info, bool with_views) {
  size_t argc = 4;
  napi_value argv[4];
  NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
  ht_ctx *ctx = Ctx(env, argv[0]);
  uint32_t n = 0;
  int32_t dw, dh;
  NAPI_OK(napi_get_array_length(env, argv[1], &n));
  napi_get_value_int32(env, argv[2], &dw); napi_get_value_int32(env, argv[3], &dh);
  if (n == 0 || dw <= 0 || dh <= 0) return Throw(env, ctx, HT_ERR_ARG);
  std::vector<ht_yuv_image> imgs(n);
  std::vector<ht_video_view> views(n);
  for (uint32_t b = 0; b < n; ++b) {
    napi_value r;
    NAPI_OK(napi_get_element(env, argv[1], b, &r));
    if (!YuvImageOf(env, r, &imgs[b]) || !ViewOf(env, r, &views[b])) return Throw(env, ctx, HT_ERR_ARG);
  }
  void *data; napi_value ab, ta;
  NAPI_OK(napi_create_arraybuffer(env, (size_t)n * dw * dh * 4, &data, &ab));
  int rc = with_views ? ht_ingest_yuv_views(ctx, imgs.data(), views.data(), (int)n, 0, static_cast<uint8_t *>(data), dw, dh)
                      : ht_ingest_yuv(ctx, imgs.data(), (int)n, 0, static_cast<uint8_t *>(data), dw, dh);
  if (rc < 0) return Throw(env, ctx, rc);
  NAPI_OK(napi_create_typedarray(env, napi_uint8_clamped_array, (size_t)n * dw * dh * 4, ab, 0, &ta));
  return ta;
}

static napi_value IngestYuv(napi_env env, napi_callback_info info) { return IngestYuvAny(env, info, false); }
static napi_value IngestYuvViews(napi_env env, napi_callback_info info) { return IngestYuvAny(env, info, true); }

// ingestViews(handle, [{width, height, rgba, view}], dw, dh) -> Uint8ClampedArray (n canvases)   (ht_ingest_views)
static napi_value IngestViews(napi_env env, napi_callback_info info) {
  size_t argc = 4;
  napi_value argv[4];
  NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
  ht_ctx *ctx = Ctx(env, argv[0]);
  uint32_t n = 0;
  int32_t dw, dh;
  NAPI_OK(napi_get_array_length(env, argv[1], &n));
  napi_get_value_int32(env, argv[2], &dw); napi_get_value_int32(env, argv[3], &dh);
  if (n == 0 || dw <= 0 || dh <= 0) return Throw(env, ctx, HT_ERR_ARG);
  std::vector<ht_video_frame> frames(n);
  std::vector<ht_video_view> views(n);
  for (uint32_t b = 0; b < n; ++b) {
    napi_value r, v;
    NAPI_OK(napi_get_element(env, argv[1], b, &r));
    std::memset(&frames[b], 0, sizeof(frames[b]));
    ht_video_frame &f = frames[b];
    f.width = (int32_t)GetNumProp(env, r, "width", 0);
    f.height = (int32_t)GetNumProp(env, r, "height", 0);
    uint8_t *rgba; size_t len;
    NAPI_OK(napi_get_named_property(env, r, "rgba", &v));
    if (!GetBytes(env, v, &rgba, &len) || len < (size_t)f.width * f.height * 4 || !ViewOf(env, r, &views[b]))
      return Throw(env, ctx, HT_ERR_ARG);
    f.rgba = rgba;
  }
  void *data; napi_value ab, ta;
  NAPI_OK(napi_create_arraybuffer(env, (size_t)n * dw * dh * 4, &data, &ab));
  int rc = ht_ingest_views(ctx, frames.data(), views.data(), (int)n, 0, static_cast<uint8_t *>(data), dw, dh);
  if (rc < 0) return Throw(env, ctx, rc);
  NAPI_OK(napi_create_typedarray(env, napi_uint8_clamped_array, (size_t)n * dw * dh * 4, ab, 0, &ta));
  return ta;
}

static napi_value Init(napi_env env, napi_value exports) {
  napi_property_descriptor d[] = {
      {"trackerConfig", nullptr, TrackerConfig, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"trackerReset", nullptr, TrackerReset, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"trackerStart", nullptr, TrackerStart, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"trackerStop", nullptr, TrackerStop, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"trackerStep", nullptr, TrackerStep, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"trackerSetParams", nullptr, TrackerSetParams, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"trackerSetDebug", nullptr, TrackerSetDebug, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"trackerSetDebugStrokes", nullptr, TrackerSetDebugStrokes, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"trackerSetFaceCrop", nullptr, TrackerSetFaceCrop, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"trackerSetFaceCropYuv", nullptr, TrackerSetFaceCropYuv, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"trackerSetFaceTensor", nullptr, TrackerSetFaceTensor, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"trackerSetCamera", nullptr, TrackerSetCamera, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"trackerSetFraming", nullptr, TrackerSetFraming, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"trackerSetRedact", nullptr, TrackerSetRedact, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"trackerSetBestShot", nullptr, TrackerSetBestShot, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"trackerExport", nullptr, TrackerExport, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"trackerImport", nullptr, TrackerImport, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"trackerFeed", nullptr, TrackerFeed, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"trackerFeedYuv", nullptr, TrackerFeedYuv, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"ingestYuv", nullptr, IngestYuv, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"trackerFeedViews", nullptr, TrackerFeedViews, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"trackerFeedYuvViews", nullptr, TrackerFeedYuvViews, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"ingestViews", nullptr, IngestViews, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"ingestYuvViews", nullptr, IngestYuvViews, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"create", nullptr, Create, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"detect", nullptr, Detect, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"trackInit", nullptr, TrackInit, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"track", nullptr, Track, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"streamStep", nullptr, StreamStep, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"streamReset", nullptr, StreamReset, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"streamHeadConfig", nullptr, StreamHeadConfig, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"streamStepHead", nullptr, StreamStepHead, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"ingest", nullptr, Ingest, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"whitebalance", nullptr, Whitebalance, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"backprojection", nullptr, Backprojection, nullptr, nullptr, nullptr, napi_default, nullptr},
  };
  napi_define_properties(env, exports, sizeof(d) / sizeof(d[0]), d);
  return exports;
}

NAPI_MODULE(NODE_GYP_MODULE_NAME, Init)
