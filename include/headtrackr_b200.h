/*
 * headtrackr_b200.h — C ABI of libheadtrackr_b200.so: the H100-native (sm_90a) replacement for
 * headtrackr's per-frame detect-then-track pixel kernels.
 *
 * This is the drop-in boundary (SURVEY.md §8b).  Every entry point replaces a call that
 * headtrackr's facetrackr.js makes into ccv.js / camshift.js / whitebalance.js; a Node N-API addon
 * (js/addon.cc) or any FFI (ctypes: headtrackr_b200/_lib.py) binds these 1:1.  Plain pointers and
 * sizes only; no C++/torch types.  All citations are into /root/reference/.
 *
 *   reference call (file:line)                                       ->  C ABI
 *   ---------------------------------------------------------------      ---------------------------
 *   headtrackr.ccv.detect_objects(headtrackr.ccv.grayscale(canvas),
 *       headtrackr.cascade, 5, 1)          src/facetrackr.js:147-149 ->  ht_detect
 *       (= src/ccv.js:22-32 grayscale + src/ccv.js:109-333 detect_objects)
 *   headtrackr.cascade                     src/cascade.js:19         ->  cascade blob given to ht_create
 *   new headtrackr.camshift.Tracker({calcAngles})
 *                                          src/facetrackr.js:64      ->  tracker slots inside ht_ctx
 *   cstracker.initTracker(canvas, Rectangle)
 *                                          src/facetrackr.js:101-107 ->  ht_track_init / ht_track_init_from_detect
 *       (= src/camshift.js:198-211)
 *   cstracker.track(canvas); getTrackObj() src/facetrackr.js:190-191 ->  ht_track
 *       (= src/camshift.js:213-312, 167-170)
 *   cstracker.getSearchWindow()            src/camshift.js:162-165   ->  ht_track (out_windows)
 *   cstracker.getBackProjectionImg()       src/facetrackr.js:195     ->  ht_backprojection
 *   headtrackr.getWhitebalance(canvas)     src/facetrackr.js:223     ->  ht_whitebalance
 *       (= src/whitebalance.js:5-29)
 *
 * Conventions
 *   - A "canvas" is a tightly packed RGBA8 frame: w*h*4 bytes, row-major (what getImageData returns).
 *     Frame batches are n contiguous frames.  `rgba` and all out pointers may be HOST or DEVICE
 *     pointers (resolved with cudaPointerGetAttributes).  With device outputs the call only enqueues
 *     work on the context's stream (use ht_sync); with host outputs it returns after the results
 *     have landed.
 *   - Return value: 0 = ok; >0 = completed with a warning (HT_WARN_*); <0 = error (HT_ERR_*).
 *     ht_last_error(ctx) describes the last non-zero return.  Nothing throws across the ABI.
 *   - One context per host thread / GPU; calls on one context must be serialised by the caller
 *     (the reference is single-threaded, src/main.js:303).
 *   - There is NO CPU fallback: every entry point fails with HT_ERR_CUDA when no sm_90 device is usable.
 */
#ifndef HEADTRACKR_B200_H
#define HEADTRACKR_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define HT_OK 0
#define HT_WARN_OVERFLOW 1      /* a per-frame raw or result list hit its capacity; lists were truncated */
#define HT_ERR_ARG (-1)
#define HT_ERR_CUDA (-2)
#define HT_ERR_SIZE (-3)        /* frame too small/large for the pyramid (a browser would throw on a 0-sized level) */
#define HT_ERR_CASCADE (-4)
#define HT_ERR_STATE (-5)       /* e.g. ht_track on a slot that was never initialised */

typedef struct ht_ctx ht_ctx;

/* One element of the array detect_objects returns (src/ccv.js:228-233 raw, :297-302 grouped):
 * x,y = top-left, all Numbers (fp64).  For raw lists (min_neighbors <= 0) neighbors == 1. */
typedef struct {
  double x, y, width, height, confidence;
  int32_t neighbors;
  int32_t pad_;
} ht_rect;

/* camshift TrackObj (src/camshift.js:362-377): x,y = centre. */
typedef struct {
  int32_t x, y, width, height;
  double angle;
} ht_trackobj;

/* camshift _searchWindow (src/camshift.js:156) */
typedef struct {
  int32_t x, y, width, height;
} ht_window;

typedef struct {
  int32_t device;             /* CUDA device ordinal */
  int32_t max_width;          /* largest frame the context must handle.  Detection has its own limit, whatever the
                               * maximum: every pyramid resample job divides by 4*dw*dh with a 32-bit multiplier,
                               * which needs dw*dh <= 2,968,721 for the largest job (W/s x H/s, s = 2^(1/(interval+1))).
                               * Largest accepted 16:9 frame before the first rejected one: 2579x1450 at interval 5,
                               * 2732x1536 at 3, 2895x1628 at 2, 3249x1827 at 1; 3840x2160 is rejected at every
                               * interval (see ht_detect).  The reference has no such limit. */
  int32_t max_height;
  int32_t max_frames;         /* largest batch per call == number of tracker slots */
  int32_t max_raw_per_frame;  /* capacity of the pre-grouping list per frame (0 -> 1024).  A crowded 640x480 frame
                               * already has more raw windows than 1024 (about 1,900 for a grid of 28 px faces).  On
                               * overflow the call returns HT_WARN_OVERFLOW and groups a subset of the windows: which
                               * subset depends on the cascade's arrival order, so the grouped list and the face the
                               * VJ->CS hand-offs pick match the reference only when the raw list did not overflow. */
  int32_t max_rects_per_frame;/* K: capacity of the result list per frame (0 -> 64).  K bounds only the list copied out
                               * (the reference's first K entries, HT_WARN_OVERFLOW when longer): the VJ->CS hand-offs
                               * of ht_detect_track, ht_stream_step(_head), ht_tracker_step and ht_tracker_feed pick the
                               * first maximum of the WHOLE grouped list, as src/facetrackr.js:157-165 does. */
  void *cuda_stream;          /* cudaStream_t to run on; NULL -> the context creates its own */
} ht_config;

/* Library/ABI version (major<<16 | minor). */
uint32_t ht_version(void);

/* cascade_blob: "HTC1" blob (tools/pack_cascade.py) of headtrackr.cascade (src/cascade.js:19). */
int ht_create(ht_ctx **out, const ht_config *cfg, const void *cascade_blob, size_t blob_len);
void ht_destroy(ht_ctx *ctx);
const char *ht_last_error(const ht_ctx *ctx);   /* ctx may be NULL: error of the last failed ht_create */
int ht_sync(ht_ctx *ctx);
int ht_max_rects(const ht_ctx *ctx);            /* K */

/* ccv.detect_objects(ccv.grayscale(frame), cascade, interval, min_neighbors) for n frames.
 *   out_rects : [n][K] ht_rect, reference order (src/ccv.js:293-330; raw order (scale,q,y,x) if min_neighbors<=0)
 *   out_counts: [n]    number of rects written for each frame
 * The input frames are not modified (the reference works on a copy, src/facetrackr.js:140-145).
 * HT_ERR_SIZE, before any kernel is launched, for a frame above max_width x max_height, for one whose pyramid has a
 * 0-sized level (the smallest frames: 81x81 at interval 5, 77x77 at 3, 64x64 at 1 and 2; a browser throws there), and
 * for one above the planner's size limit ("frame too large for 32-bit bilinear numerators").  That limit: k_resample
 * computes floor(n / (4*dw*dh)) as (n * M) >> k with n and M 32-bit; the numerator n <= 1022*dw*dh fits up to
 * dw*dh = 4,202,512, but the multiplier M (between n_max and 2*n_max) only up to dw*dh = 2,968,721, and again in
 * 4,194,305..4,198,406.  So the largest accepted 16:9 frames are 2579x1450 at interval 5 (2580x1451 is rejected),
 * 2732x1536 at 3, 2895x1628 at 2 and 3249x1827 at 1 (beyond those, a few isolated sizes are accepted again, such as
 * 3864x2173 at 1); 3840x2160 is rejected at every interval.  The reference has no such limit: it detects at
 * 2580x1451 and 3840x2160 too.  The same limit applies to every entry point that detects. */
int ht_detect(ht_ctx *ctx, const uint8_t *rgba, int n, int w, int h, int interval, int min_neighbors,
              ht_rect *out_rects, int32_t *out_counts);

/* camshift.Tracker.initTracker(frame, Rectangle(x,y,w,h)) for n tracker slots (src/camshift.js:198-211).
 *   slots : [n] DISTINCT slot ids in [0,max_frames) (NULL -> 0..n-1); rgba: n frames; rects: [n][4] = x,y,w,h
 *           (host arrays are checked: out-of-range or repeated ids -> HT_ERR_ARG; a device-resident slot array is
 *           used as is - ids out of range or repeated are undefined behaviour, like any bad device pointer)
 * Pixels of the rectangle outside the frame count as (0,0,0) like canvas getImageData. */
int ht_track_init(ht_ctx *ctx, const int32_t *slots, int n, const uint8_t *rgba, int w, int h,
                  const int32_t *rects, int calc_angles);

/* The VJ->CS hand-off of facetrackr (src/facetrackr.js:157-165 first-max-confidence pick, :97-108
 * confidence > -10 gate and Math.floor of x,y,w,h) done on the device from ht_detect's outputs:
 *   det_rects [n][K], det_counts [n] (host or device).  out_found [n] (optional): 1 if the slot was seeded.
 * The pick is over the list passed in: det_rects[k][0, min(det_counts[k], K)).  When ht_detect truncated a list to K
 * entries, the pick can differ from the reference's; ht_detect_track picks from the whole list. */
int ht_track_init_from_detect(ht_ctx *ctx, const int32_t *slots, int n, const uint8_t *rgba, int w, int h,
                              const ht_rect *det_rects, const int32_t *det_counts, int calc_angles,
                              int32_t *out_found);

/* n_calls successive camshift.Tracker.track(frame) calls on each slot's frame, state carried
 * (src/camshift.js:213-312).  out_objs [n] = getTrackObj() after the last call; out_windows [n]
 * (optional) = getSearchWindow().  Slots that were never initialised yield HT_ERR_STATE. */
int ht_track(ht_ctx *ctx, const int32_t *slots, int n, const uint8_t *rgba, int w, int h, int n_calls,
             ht_trackobj *out_objs, ht_window *out_windows);

/* One facetrackr VJ frame followed by its CS frames, for a batch (src/facetrackr.js:67-126):
 *   ht_detect -> first-max-confidence pick, confidence > -10 gate, floor -> initTracker on slot k for frame k
 *   -> n_calls x track().  Frames with no usable face leave out_found[k] = 0 and a zero TrackObj.
 * The pick is over the whole grouped list, also when out_rects holds only its first K entries (HT_WARN_OVERFLOW).
 * With HOST frames the upload is pipelined in chunks against the kernels of the previous chunk.
 * out_found and out_windows are optional. */
int ht_detect_track(ht_ctx *ctx, const uint8_t *rgba, int n, int w, int h, int interval, int min_neighbors,
                    int calc_angles, int n_calls, ht_rect *out_rects, int32_t *out_counts, int32_t *out_found,
                    ht_trackobj *out_objs, ht_window *out_windows);

/* facetrackr's per-frame state machine for n independent video streams, on the device (SURVEY.md 8f-2).
 * Stream k (tracker slot k) is in one of the reference's detection modes (src/facetrackr.js:57,75-81; whitebalancing
 * off, as after src/main.js:236):
 *   "VJ": ccv.detect_objects on the frame, first-max-confidence pick (src/facetrackr.js:157-165); if its confidence
 *         exceeds -10 the tracker is seeded with the floored rectangle on this same frame and the stream switches
 *         to "CS" (src/facetrackr.js:97-108)
 *   "CS": one camshift track() on the frame (src/facetrackr.js:178-209); a result with width or height 0 means the
 *         face is lost and the stream starts over in "VJ" on the next frame (src/main.js:230-244, retryDetection)
 * ht_stream_step consumes ONE frame per stream (rgba = n frames, stream-major) and returns the TrackObj facetrackr
 * would hold after track() for each stream; the host emits `facetrackingEvent` for records with detection == 2
 * (src/facetrackr.js:112-125).  Mode switches, the pick and the tracker seeding happen in kernels: the only host
 * traffic per frame is the frame upload (if `rgba` is host memory) and the n event records. */
typedef struct {
  int32_t detection;   /* 1 = "VJ", 2 = "CS" */
  int32_t status;      /* bit 0: face found on this frame (VJ -> CS); bit 1: face lost on this frame (CS -> VJ) */
  double x, y, width, height, angle, confidence;   /* VJ: top-left, fp64 as ccv returns; CS: centre, integers */
} ht_stream_event;
/* Head position per stream and frame as an epilogue of the state machine (SURVEY.md 8f-3): what src/main.js does
 * with a "CS" result - headtrackrStatus "found" (src/main.js:246-249), headtrackr.Smoother (src/smoother.js:25-87,
 * including its quirks: sp2 aliases sp, z is NaN, predict() runs with step 0), the wait for six head diagonals within
 * 5 px (src/main.js:262-281), headposition.Tracker with its field-of-view estimate and edge correction
 * (src/headposition.js:35-191) - evaluated by the kernel that already writes the stream events.  One ht_head_event
 * per stream and frame; `valid` marks the frames on which the reference dispatches `headtrackingEvent {x, y, z}`. */
typedef struct {
  int32_t smoothing;           /* params.smoothing      (src/main.js:39, default 1) */
  int32_t head_position;       /* params.headPosition   (src/main.js:55, default 1) */
  int32_t edgecorrection;      /* headposition params   (src/headposition.js:44-48, default 1) */
  int32_t pad_;
  double alpha;                /* Smoother alpha        (src/main.js:163: 0.35) */
  double fov_deg;              /* params.fov in degrees; <= 0: estimate it from the first stable face (src/main.js:283-288) */
  double camera_offset;        /* params.cameraOffset   (src/main.js:53: 11.5) */
  double distance_to_screen;   /* 60 cm                 (src/headposition.js:75-79) */
} ht_head_params;
typedef struct {
  int32_t valid;               /* 1: headtrackingEvent dispatched on this frame */
  int32_t status;              /* bit 0: headtrackrStatus "found" on this frame */
  double x, y, z;              /* head position in cm relative to the screen centre (src/headposition.js:165-188) */
  double fx, fy, fwidth, fheight;   /* the (smoothed) face object it was computed from */
} ht_head_event;
/* params == NULL switches the epilogue off.  Changing parameters does not reset stream state; ht_stream_reset does. */
int ht_stream_head_config(ht_ctx *ctx, const ht_head_params *params);
/* ht_stream_step plus one ht_head_event per stream (out_head may be NULL) */
int ht_stream_step_head(ht_ctx *ctx, const uint8_t *rgba, int n, int w, int h, int interval, int min_neighbors,
                        int calc_angles, ht_stream_event *out_events, ht_head_event *out_head);

/* put streams [first, first+n) back into "VJ" (new facetrackr.Tracker) */
int ht_stream_reset(ht_ctx *ctx, int first, int n);
/* The "VJ" pick is over the whole grouped list of the stream's frame: K (max_rects_per_frame) does not change which
 * face is tracked.  A frame whose raw list overflows max_raw_per_frame returns HT_WARN_OVERFLOW, and its pick may differ
 * from the reference's. */
int ht_stream_step(ht_ctx *ctx, const uint8_t *rgba, int n, int w, int h, int interval, int min_neighbors,
                   int calc_angles, ht_stream_event *out_events);

/* headtrackr.Tracker per stream on the device from its first frame (SURVEY.md 8f-5, ABI 1.1): what src/main.js does
 * between start() and stop() - the starter's content check (src/main.js:307-326: a frame whose getWhitebalance is 0
 * is retried on the next frame), facetrackr with whitebalancing (src/facetrackr.js:42-52,79-95: 15 whitebalance
 * samples within 2 gray levels before detection starts), VJ -> CS, the headtrackrStatus events, the lost face with or
 * without retryDetection, and the head-position epilogue of ht_stream_step_head.  Stream k uses tracker slot k.
 * Per stream the mode is one of IDLE (not running: its frame is never read), STARTING, WB, VJ, CS; one
 * ht_tracker_step call is one timer tick of streams [0, n) (ht_tracker_feed: of any subset, each with its own video
 * and clock).  Detection runs with interval 5 and min_neighbors 1
 * (src/facetrackr.js:147-149).
 * While the lifecycle is configured ht_stream_step / ht_stream_step_head return HT_ERR_STATE (the two share the
 * tracker slots).  One deliberate difference: start() on a running stream does nothing, where the reference would
 * run an extra, unscheduled pass. */
typedef struct {
  int32_t retry_detection;   /* params.retryDetection (src/main.js:40, default 1) */
  int32_t calc_angles;       /* params.calcAngles     (src/main.js:54, default 0) */
  int32_t pad_[2];
  ht_head_params head;       /* smoothing, headPosition, fov, cameraOffset: as for ht_stream_head_config */
} ht_tracker_params;
/* headtrackrStatus events of one frame: bit order == dispatch order (src/main.js:182,183,193,233,246,350,251) */
#define HT_STATUS_WHITEBALANCE 1
#define HT_STATUS_DETECTING 2
#define HT_STATUS_HINTS 4
#define HT_STATUS_REDETECTING 8
#define HT_STATUS_LOST 16
#define HT_STATUS_STOPPED 32     /* the stop() of a lost face without retryDetection; ht_tracker_stop emits none */
#define HT_STATUS_FOUND 64
/* One record per stream and frame.  Dispatch order of the reference: `facetrackingEvent` (detection == 2) first, then
 * the status bits from low to high, then `headtrackingEvent` (head.valid).  status "tracking" is set without an
 * event on every "CS" frame before its redetecting / lost / found (src/main.js:227). */
typedef struct {
  int32_t detection;         /* 0 = no pass ran (idle, or the starter saw no content), 1 = "VJ", 2 = "CS", 3 = "WB" */
  int32_t status;            /* HT_STATUS_* */
  double x, y, width, height, angle, confidence;   /* facetrackr TrackObj (VJ: top-left; CS: centre) */
  double wb;                 /* getWhitebalance of the frame when the starter or a "WB" pass ran, else 0 */
  int32_t running;           /* 1: a track() pass is scheduled for the next frame */
  int32_t pad_;
  double fov;                /* getFOV() after this frame (src/main.js:363-365) */
  ht_head_event head;        /* smoothed face and headtrackingEvent {x, y, z} */
} ht_tracker_event;
/* params == NULL switches the lifecycle off and puts every stream back into ht_stream_reset's state.  Switching it on
 * starts every stream as ht_tracker_reset; changing parameters while on keeps the stream states. */
int ht_tracker_config(ht_ctx *ctx, const ht_tracker_params *params);
int ht_tracker_reset(ht_ctx *ctx, int first, int n);   /* new headtrackr.Tracker + init(): not running */
int ht_tracker_start(ht_ctx *ctx, int first, int n);   /* start(): the next frame of the stream goes through starter() */
int ht_tracker_stop(ht_ctx *ctx, int first, int n);    /* stop() (src/main.js:347-355); the caller emits "stopped" */
/* one frame per stream for streams [0, n): rgba = n frames, stream-major; now_ms = (new Date).getTime() of this tick
 * (the "hints" timer, src/main.js:187-194); out[n] host or device (device: enqueue only) */
int ht_tracker_step(ht_ctx *ctx, const uint8_t *rgba, int n, int w, int h, double now_ms, ht_tracker_event *out);

/* One stream's video frame for ht_tracker_feed (ABI 1.2). */
typedef struct {
  const uint8_t *rgba;    /* the stream's video frame: RGBA8, `height` rows of `pitch` bytes */
  int32_t stream;         /* tracker stream id in [0, max_frames) */
  int32_t width, height;  /* video size, 1..16384 */
  int32_t pitch;          /* bytes per row; 0 -> 4*width; a multiple of 4 and >= 4*width */
  double now_ms;          /* (new Date).getTime() when this stream's timer fired */
} ht_video_frame;         /* 32 bytes */
/* One timer tick of each listed stream, each on its own video and clock: drawImage(video, 0, 0, canvas_w, canvas_h)
 * (src/main.js:170, 312; the canvas resampler of ht_ingest) followed by exactly what ht_tracker_step does for that
 * stream - a track() pass (src/main.js:168-305) or the starter (src/main.js:307-326).  Cameras tick independently, so
 * any subset of the streams may be listed, in any order; streams that are not listed do not tick and their state does
 * not change.  A listed IDLE stream yields ht_tracker_step's IDLE record and its video is neither read nor drawn.
 *   frames: n HOST records with distinct stream ids.  Their pixel pointers are all device memory (frames_on_device
 *           = 1) or all host memory (0: the library uploads them); only the first record's pointer is checked.
 *   canvas_w x canvas_h: the working canvas of every record of the call (it sets the pyramid plan), at most
 *           max_width x max_height.  The library draws into its own canvas arena ([max_frames] canvases, allocated at
 *           the first call).
 *   out[n]: one ht_tracker_event per record, in record order; host or device (device: enqueue only).
 * Errors (nothing is enqueued): HT_ERR_STATE without ht_tracker_config; HT_ERR_ARG for n outside [1, max_frames], a
 * stream id out of range or listed twice, a NULL pixel pointer, a pointer or pitch that is not a multiple of 4, a
 * pitch below 4*width, or a first pointer whose memory space contradicts frames_on_device; HT_ERR_SIZE for a video
 * size outside 1..16384 or a canvas that is 0-sized, larger than max_width x max_height or too small for the pyramid.
 * ht_tracker_step and ht_tracker_feed may be mixed on one context: both tick the same per-stream state.  In both, the
 * "VJ" pick is over the whole grouped list (as for ht_stream_step), unless the raw list overflowed (HT_WARN_OVERFLOW). */
int ht_tracker_feed(ht_ctx *ctx, const ht_video_frame *frames, int n, int frames_on_device, int canvas_w, int canvas_h,
                    ht_tracker_event *out);

/* Frame ingest (SURVEY.md 8f-4): canvasContext.drawImage(videoElement, 0, 0, canvas.width, canvas.height)
 * (src/main.js:170) for n frames - the video frame (sw x sh) scaled onto the working canvas (dw x dh), all four
 * channels, with the canvas resampler this build defines (DESIGN.md 2).  src and dst may be host or device
 * memory; a device dst can be passed straight to ht_detect / ht_track / ht_stream_step.  (The 1:1 copy facetrackr
 * makes before detection, src/facetrackr.js:140-145, needs no call: no entry point modifies its input frames.) */
int ht_ingest(ht_ctx *ctx, const uint8_t *src_rgba, int n, int sw, int sh, uint8_t *dst_rgba, int dw, int dh);

/* getBackProjectionImg() of the last track() state for one slot: RGBA w*h*4, floor(255*weight) gray
 * (src/camshift.js:177-196).  Debug path of the reference (src/facetrackr.js:194-196). */
int ht_backprojection(ht_ctx *ctx, int slot, const uint8_t *rgba, int w, int h, uint8_t *out_rgba);

/* headtrackr.getWhitebalance(frame) for n frames: out[n] doubles (src/whitebalance.js:5-29). */
int ht_whitebalance(ht_ctx *ctx, const uint8_t *rgba, int n, int w, int h, double *out);

/* ---- introspection used by the parity tests (not needed by a caller of the reference API) ---- */

/* pyramid geometry for (w,h,interval): n_slots, scale_upto and the per-slot sizes (src/ccv.js:110-127) */
int ht_plan_info(ht_ctx *ctx, int w, int h, int interval, int32_t *n_slots, int32_t *scale_upto,
                 int32_t *slot_w, int32_t *slot_h, int cap);
/* copy one pyramid plane (slot, q) of frame `frame` of the LAST ht_detect call to host memory (w*h bytes) */
int ht_debug_plane(ht_ctx *ctx, int frame, int slot, int q, uint8_t *out, int cap_bytes, int32_t *w, int32_t *h);
/* raw (pre-grouping) list of frame `frame` of the LAST ht_detect call, reference order */
int ht_debug_raw(ht_ctx *ctx, int frame, ht_rect *out, int cap, int32_t *count);
/* tracker slot state: model histogram (4096 u32, optional) */
int ht_debug_model_hist(ht_ctx *ctx, int slot, uint32_t *out4096);
/* mean-shift counters since the last reset: {moment passes summed on the device, passes redone in strict reference
 * order, window pixels visited, track() calls, passes answered from the per-launch window memo} */
int ht_debug_track_stats(ht_ctx *ctx, uint64_t *out5, int reset);
/* Exactness fallbacks (tests only).  The kernels decide the integer outputs of the reference exactly with cheap
 * arithmetic plus a fallback that reproduces the reference's own operation order when the cheap path is not
 * conclusive.  flags force the fallbacks so that they are exercised (results must not change):
 *   bit 0: every generated cascade-stage decision of the survivor lists is treated as an exact tie and re-decided
 *          with ordered fp64 adds (src/ccv.js:186-222)
 *   bit 1: the same for the late (warp-per-window, exact-integer) stages
 *   bit 2: every mean-shift pass of ht_track re-derives its moments in the reference's strict summation order
 *          (src/camshift.js:90-107) as if a truncation had been ambiguous */
int ht_debug_set_exactness(ht_ctx *ctx, int flags);
/* Window memo of ht_track / ht_detect_track (default on).  The moments of a search window depend only on the frame,
 * the histogram weights and the window, and all three are fixed for the n_calls track() calls of one launch; the
 * kernel therefore keeps the moments of the last 8 windows of a stream and re-uses them when mean-shift comes back
 * to one of them (a converged stream; a stream oscillating between two windows - src/camshift.js:283-306 would
 * re-sum them).  Results are identical either way; enable = 0 re-sums every pass like the reference. */
int ht_set_track_memo(ht_ctx *ctx, int enable);
/* Pipelined batches (default off; HT_PIPELINE=1 in the environment turns it on at ht_create).  With enable != 0 an
 * ht_detect_track call whose frames AND outputs are all device pointers returns as soon as its detection is enqueued
 * and leaves its tracking (hand-off + n_calls x track(), src/facetrackr.js:97-108,190) on a second, higher-priority
 * stream, where it runs under the detection kernels of the NEXT ht_detect_track call: CAMShift is a latency chain per
 * stream that leaves most of the GPU idle, the detector is throughput-bound.  Results are identical to the
 * unpipelined call.  The caller's side of the contract: out_found / out_objs / out_windows of call s are complete
 * after ht_sync or ht_join (or any other entry point of the context, which all join first) - NOT merely after the
 * next ht_detect_track; out_rects / out_counts may be reused by the next call (the library orders the accesses);
 * the frames of call s must stay unchanged until then as well. */
int ht_set_pipeline(ht_ctx *ctx, int enable);
/* Stream-level join: later work on the context's stream waits for a pipelined call's tracking.  No host wait. */
int ht_join(ht_ctx *ctx);
/* per-stream timeline of the last ht_track / ht_detect_track launch, 4 x u64 per stream: {globaltimer ns at start,
 * at end, SM id of the leading CTA, moment passes}.  Only for contexts created with HT_TRACK_TRACE=1 in the
 * environment (tools/track_timeline.py); HT_ERR_ARG otherwise. */
int ht_debug_track_trace(ht_ctx *ctx, uint64_t *out, int n_streams);
/* profiling builds (-DHT_TRACK_PASSTRACE=1) only, zeros otherwise: 8 x u64 per stream, the SM clock cycles the leading
 * thread spent in each phase of its passes {pixel loop, warp sums + CTA barrier, exchange + cluster barrier, scalar
 * mean-shift step, publishing barrier, 0, 0, 0}, summed over the launch. */
int ht_debug_track_phases(ht_ctx *ctx, uint64_t *out, int n_streams);
/* number of kernels this context has launched so far (bench.py's gpu_launches) */
uint64_t ht_launch_count(const ht_ctx *ctx);

/* Per-kernel-class device time, measured with CUDA events recorded on the context's stream around
 * every launch while enabled (bench.py's roofline uses the cascade class).  ht_profile_read syncs the
 * stream and returns the accumulated milliseconds and launch counts per class. */
enum { HT_PROF_GRAY = 0, HT_PROF_PYRAMID, HT_PROF_CASCADE, HT_PROF_GROUP, HT_PROF_HIST, HT_PROF_TRACK_INIT,
       HT_PROF_TRACK, HT_PROF_N };
int ht_profile(ht_ctx *ctx, int enable);
int ht_profile_read(ht_ctx *ctx, double *ms_out, uint64_t *launches_out, int reset);

#ifdef __cplusplus
}
#endif
#endif
