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
 * starts every stream as ht_tracker_reset; changing parameters while on keeps the stream states.  Either way every
 * stream gets `params`: per-stream values of ht_tracker_set_params are discarded, and so are the debug canvases of
 * ht_tracker_set_debug. */
int ht_tracker_config(ht_ctx *ctx, const ht_tracker_params *params);
/* Per-stream parameters (ABI 1.3): stream first+i gets params[i] (host), for i in [0, n) - the parameters of its own
 * `new headtrackr.Tracker(params)`.  Stream states are kept, as when ht_tracker_config changes parameters while on.
 * calc_angles takes effect at the stream's next hand-off to camshift (initTracker: facetrackr creates its camshift
 * tracker with it, src/main.js:173,241); every other field on the stream's next tick.
 * Errors (nothing changes): HT_ERR_STATE before ht_tracker_config; HT_ERR_ARG for a range outside [0, max_frames),
 * n <= 0, params NULL, or any record ht_tracker_config would reject (alpha outside [0,1], distance_to_screen <= 0). */
int ht_tracker_set_params(ht_ctx *ctx, int first, int n, const ht_tracker_params *params);
int ht_tracker_reset(ht_ctx *ctx, int first, int n);   /* new headtrackr.Tracker + init(): not running */
int ht_tracker_start(ht_ctx *ctx, int first, int n);   /* start(): the next frame of the stream goes through starter() */
int ht_tracker_stop(ht_ctx *ctx, int first, int n);    /* stop() (src/main.js:347-355); the caller emits "stopped" */
/* one frame per stream for streams [0, n): rgba = n frames, stream-major; now_ms = (new Date).getTime() of this tick
 * (the "hints" timer, src/main.js:187-194); out[n] host or device (device: enqueue only).  While one of the streams
 * has a face redaction (ht_tracker_set_redact) the library writes the frames in place, and they must be device
 * memory (HT_ERR_ARG otherwise, nothing enqueued). */
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
 *           max_width x max_height.  The library draws into its own canvas arena (at least [max_frames] canvases of
 *           the call's largest size, grown and zeroed when a call needs more).  This is ht_tracker_feed_canvases with
 *           every record on canvas_w x canvas_h.
 *   out[n]: one ht_tracker_event per record, in record order; host or device (device: enqueue only).
 * Errors (nothing is enqueued): HT_ERR_STATE without ht_tracker_config; HT_ERR_ARG for n outside [1, max_frames], a
 * stream id out of range or listed twice, a NULL pixel pointer, a pointer or pitch that is not a multiple of 4, a
 * pitch below 4*width, or a first pointer whose memory space contradicts frames_on_device; HT_ERR_SIZE for a video
 * size outside 1..16384 or a canvas that is 0-sized, larger than max_width x max_height or too small for the pyramid.
 * A record whose stream has a face redaction (ht_tracker_set_redact) must have device video that shares no byte with
 * another redacting record's; the library writes it in place (HT_ERR_ARG otherwise, nothing enqueued).
 * ht_tracker_step and ht_tracker_feed may be mixed on one context: both tick the same per-stream state.  In both, the
 * "VJ" pick is over the whole grouped list (as for ht_stream_step), unless the raw list overflowed (HT_WARN_OVERFLOW). */
int ht_tracker_feed(ht_ctx *ctx, const ht_video_frame *frames, int n, int frames_on_device, int canvas_w, int canvas_h,
                    ht_tracker_event *out);

/* One stream's video frame and working canvas for ht_tracker_feed_canvases (ABI 1.3): in the reference each
 * headtrackr.Tracker draws onto its own canvas, whose size also feeds headposition (src/main.js:170, 284-291). */
typedef struct {
  ht_video_frame video;
  int32_t canvas_w, canvas_h;   /* this record's working canvas */
  int32_t pad_[2];
} ht_canvas_frame;              /* 48 bytes */
/* ht_tracker_feed with a canvas per record; the same contract otherwise (any subset of streams in any order, host or
 * device videos, out[n] in record order, everything checked before anything is enqueued).  Records on different
 * canvas sizes tick in the same call: the library groups them by size and runs the detector and camshift once per
 * size, every per-stream kernel once per call.  A record gives the same canvas and the same event whatever else is in
 * the call.  Errors as for ht_tracker_feed; a record's canvas that is 0-sized, larger than max_width x max_height, too
 * small for the pyramid or too large for the resampler is HT_ERR_SIZE with the record's index in ht_last_error. */
int ht_tracker_feed_canvases(ht_ctx *ctx, const ht_canvas_frame *frames, int n, int frames_on_device,
                             ht_tracker_event *out);

/* Video as decoders, cameras and capture APIs write it.  The frame is drawn as the RGBA8 frame this library's
 * conversion makes of it (DESIGN.md 2, "YUV video"): luma pixel (x, y) takes chroma sample (x >> sx, y >> sy) of its
 * format, then an integer BT.601, BT.709 or BT.2020 matrix, limited or full range, A = 255; the packed RGB formats are
 * taken as they are.  Byte offsets:
 *     0  const uint8_t *planes[3]   per format, below; a plane the format does not use must be NULL
 *    24  int32 pitch[3]             bytes per row; 0 -> the tight pitch below; otherwise >= that, any alignment (P010:
 *                                   even pointers and pitches) (unused for a NULL plane)
 *    36  int32 width, height        luma size w x h, 1..16384; cw = ceil(w/2), ch = ceil(h/2)
 *    44  int32 format               one of the HT_YUV_ formats below
 *    48  int32 color                HT_YUV_BT601, HT_YUV_BT709 or HT_YUV_BT2020, optionally | HT_YUV_FULL_RANGE (not
 *                                   BT709 | BT2020); 0 for the packed RGB formats
 *    52  int32 pad_
 *  format        planes                         tight pitches   luma (x, y)      chroma / colour samples of pixel (x, y)
 *  NV12  (0)     Y, UV (U first), NULL          w, 2cw          Y[y][x]          U = UV[y>>1][2(x>>1)], V = ... + 1
 *  I420  (1)     Y, U, V                        w, cw, cw       Y[y][x]          U[y>>1][x>>1], V[y>>1][x>>1]
 *  NV21  (16)    Y, VU (V first), NULL          w, 2cw          Y[y][x]          V = VU[y>>1][2(x>>1)], U = ... + 1
 *  I422  (17)    Y, U, V (h chroma rows)        w, cw, cw       Y[y][x]          U[y][x>>1], V[y][x>>1]
 *  I444  (18)    Y, U, V                        w, w, w         Y[y][x]          U[y][x], V[y][x]
 *  YUYV  (19)    P, NULL, NULL                  4cw             P[y][2x]         U = P[y][4(x>>1)+1], V = ...+3
 *  UYVY  (20)    P, NULL, NULL                  4cw             P[y][2x+1]       U = P[y][4(x>>1)],   V = ...+2
 *  P010  (21)    Y, UV (U first), NULL:         2w, 4cw         r(Y[y][x])       U = r(UV[y>>1][2(x>>1)]),
 *                16-bit little-endian samples                                    V = r(UV[y>>1][2(x>>1)+1])
 *  BGRA  (32)    P, NULL, NULL                  4w              -                R, G, B, A = bytes 4x+2, 4x+1, 4x, 4x+3
 *  BGR24 (33)    P, NULL, NULL                  3w              -                R, G, B = bytes 3x+2, 3x+1, 3x; A = 255
 *  RGB24 (34)    P, NULL, NULL                  3w              -                R, G, B = bytes 3x, 3x+1, 3x+2; A = 255
 * P010 samples are reduced to 8 bits, r(s) = min(255, (s + 128) >> 8) of the whole 16-bit word (P016 is valid P010),
 * and then converted as 8-bit samples: a P010 frame draws exactly like the NV12 frame of its reduced samples. */
#define HT_YUV_NV12 0
#define HT_YUV_I420 1
#define HT_YUV_NV21 16
#define HT_YUV_I422 17
#define HT_YUV_I444 18
#define HT_YUV_YUYV 19
#define HT_YUV_UYVY 20
#define HT_YUV_P010 21
#define HT_YUV_BGRA 32
#define HT_YUV_BGR24 33
#define HT_YUV_RGB24 34
#define HT_YUV_BT601 0
#define HT_YUV_BT709 1
#define HT_YUV_FULL_RANGE 2
#define HT_YUV_BT2020 8
typedef struct {
  const uint8_t *planes[3];
  int32_t pitch[3];
  int32_t width, height;
  int32_t format;
  int32_t color;
  int32_t pad_;
} ht_yuv_image;           /* 56 bytes */
/* One stream's YUV video frame, working canvas and clock for ht_tracker_feed_yuv: the YUV counterpart of
 * ht_canvas_frame.  Byte offsets: 0 video, 56 stream, 60 canvas_w, 64 canvas_h, 68 pad_, 72 now_ms. */
typedef struct {
  ht_yuv_image video;
  int32_t stream;               /* tracker stream id in [0, max_frames) */
  int32_t canvas_w, canvas_h;   /* this record's working canvas */
  int32_t pad_;
  double now_ms;                /* (new Date).getTime() when this stream's timer fired */
} ht_yuv_frame;                 /* 80 bytes */
/* ht_tracker_feed_canvases on YUV video: drawImage(video, 0, 0, canvas_w, canvas_h) of the decoded frame, converted
 * and scaled in one pass straight from the planes (no RGBA copy of the video is made), then the same tick.  A record
 * gives exactly the canvas and the event of ht_tracker_feed_canvases on the RGBA8 frame the conversion makes of its
 * video.  The contract is ht_tracker_feed_canvases's: any subset of streams in any order, each record with its own
 * canvas and clock, out[n] in record order on the host or the device, an IDLE stream's planes never read.  The
 * streams' state is the one every tick uses: a stream may tick from YUV, RGBA and ht_tracker_step in turn.  Host
 * planes are packed into the library's staging buffer; only the first record's Y pointer is tested against
 * frames_on_device.  Records may mix every format, colour and canvas size.  Same launches as ht_tracker_feed_canvases
 * on the same canvases.
 * Errors (nothing is enqueued): those of ht_tracker_feed_canvases, and HT_ERR_ARG, with the record's index in
 * ht_last_error, for a format outside the values above or a color not valid for it, a NULL plane the format uses, a
 * non-NULL plane it does not use, a pitch below the tight pitch, or an odd P010 plane pointer or pitch; HT_ERR_SIZE for
 * a video size outside 1..16384. */
int ht_tracker_feed_yuv(ht_ctx *ctx, const ht_yuv_frame *frames, int n, int frames_on_device, ht_tracker_event *out);
/* ht_ingest for YUV video: src[i] (host records; planes all host or all device memory, as frames_on_device says, only
 * src[0]'s Y pointer is tested) drawn onto the i-th tightly packed dw x dh RGBA8 canvas of dst_rgba (host or device
 * memory; a 4-byte aligned pointer), for i in [0, n).  The frames may differ in size, format and color.  One launch.
 * Errors (nothing is enqueued): HT_ERR_ARG for NULL pointers, n <= 0, a misaligned dst, a contradicting memory space
 * or a bad record (as for ht_tracker_feed_yuv); HT_ERR_SIZE for sizes outside 1..16384 or a canvas too large for the
 * resampler. */
int ht_ingest_yuv(ht_ctx *ctx, const ht_yuv_image *src, int n, int frames_on_device, uint8_t *dst_rgba, int dw, int dh);

/* A view of a video frame (DESIGN.md 2, "Views"): an orientation, then a source rectangle of the oriented frame.
 * orientation & 3 rotates the w x h video V clockwise by 0, 90, 180 or 270 degrees, and HT_VIEW_MIRROR then mirrors
 * the rotated frame horizontally.  The oriented frame O is w x h (0, 180) or h x w (90, 270), and its pixel (x, y) is
 * V(x, y), V(y, h-1-x), V(w-1-x, h-1-y) or V(w-1-y, x) for 0, 90, 180, 270; with the mirror bit, O(W'-1-x, y) of that.
 * For YUV formats the orientation maps luma coordinates and chroma is looked up as the format says, so a rotated
 * frame is the rotation of its converted RGBA8 frame.  (sx, sy, sw, sh) is a rectangle of O, all 0 for the whole of
 * it, otherwise sw, sh >= 1, sx, sy >= 0, sx + sw <= W' and sy + sh <= H'.  The canvas is then drawImage(O, sx, sy, sw,
 * sh, 0, 0, canvas_w, canvas_h): taps are clamped to the rectangle, and an sw x sh rectangle on an sw x sh canvas is
 * copied.  EXIF orientations 1..8 are views 0, 4, 2, 6, 5, 1, 7, 3; a rotation r (clockwise, applied first) with a
 * horizontal flip is r / 90 | HT_VIEW_MIRROR.  Events, debug canvases and cameras stay in canvas coordinates. */
#define HT_VIEW_ROTATE_90 1
#define HT_VIEW_ROTATE_180 2
#define HT_VIEW_ROTATE_270 3
#define HT_VIEW_MIRROR 4
typedef struct {
  int32_t orientation;          /* 0..7 */
  int32_t sx, sy, sw, sh;       /* in the oriented frame; all 0 = the whole frame */
  int32_t reserved[3];          /* must be 0 */
} ht_video_view;                /* 32 bytes */
/* ht_tracker_feed_canvases with a view per record: record i's video is drawn through views[i].  The contract is
 * ht_tracker_feed_canvases's (any subset of streams, canvases of any size, host or device video, out[n] in record
 * order, the same launches); several records may point into the same device frame.  A record with the identity view
 * (orientation 0, whole frame) gives exactly the canvas and event of ht_tracker_feed_canvases.
 * Errors (nothing is enqueued): those of ht_tracker_feed_canvases, and HT_ERR_ARG for views == NULL and, with the
 * record's index in ht_last_error, for an orientation outside 0..7, a non-zero reserved field, or a rectangle that is
 * not (0, 0, 0, 0) and is empty or not inside the oriented frame. */
int ht_tracker_feed_views(ht_ctx *ctx, const ht_canvas_frame *frames, const ht_video_view *views, int n,
                          int frames_on_device, ht_tracker_event *out);
/* ht_tracker_feed_yuv with a view per record, as ht_tracker_feed_views is to ht_tracker_feed_canvases. */
int ht_tracker_feed_yuv_views(ht_ctx *ctx, const ht_yuv_frame *frames, const ht_video_view *views, int n,
                              int frames_on_device, ht_tracker_event *out);
/* ht_ingest through views: src[i] (an RGBA8 frame; its stream and now_ms are ignored) drawn through views[i] onto the
 * i-th tightly packed dw x dh canvas of dst_rgba.  The frames may differ in size.  One launch.  Errors: those of
 * ht_ingest_yuv, for RGBA8 records those of ht_tracker_feed's, and the view errors of ht_tracker_feed_views. */
int ht_ingest_views(ht_ctx *ctx, const ht_video_frame *src, const ht_video_view *views, int n, int frames_on_device,
                    uint8_t *dst_rgba, int dw, int dh);
/* ht_ingest_yuv through views, as ht_ingest_views. */
int ht_ingest_yuv_views(ht_ctx *ctx, const ht_yuv_image *src, const ht_video_view *views, int n, int frames_on_device,
                        uint8_t *dst_rgba, int dw, int dh);

/* A stream's debug canvas: `params.debug` of its headtrackr.Tracker (src/main.js:42-50). */
typedef struct {
  uint8_t *rgba;          /* DEVICE memory, `height` rows of `pitch` bytes; NULL: the stream has no debug canvas */
  int32_t width, height;  /* 1..16384 */
  int32_t pitch;          /* 0 -> 4*width; a multiple of 4, >= 4*width */
  int32_t pad_;
} ht_debug_canvas;        /* 24 bytes */
/* Stream first+i gets canvases[i] (host array), for i in [0, n); stream states are kept.  On every tick of a stream
 * whose facetrackr pass is "CS" - track() ran, including the pass that loses the face - the library does what
 * facetrackr does with params.debug (src/facetrackr.js:193-196): putImageData(getBackProjectionImg(), 0, 0).  Each
 * pixel of the working canvas becomes (v, v, v, 255), v = floor(255 * min(model[bin] / current[bin], 1)) in fp64 (0
 * where current[bin] is 0), with this frame's histogram; the image is clipped to the debug canvas, and pixels outside
 * min(w, width) x min(h, height) keep what they held.  IDLE, STARTING, WB and VJ ticks (also the VJ tick that finds a
 * face) write nothing.  The canvas is never cleared, and survives stop, start, reset and a lost face, as main.js hands
 * one params.debug to every facetrackr it creates.  The strokes main.js draws on top (src/main.js:199-219) are drawn
 * only for streams that turn them on (ht_tracker_set_debug_strokes); otherwise they are left to the caller, as pure
 * functions of the tick's ht_tracker_event (streams.debug_calls in the Python package).  The writes are enqueued on the context's stream before a tick's outputs: with host `out` they have landed when the
 * tick returns, with device `out` after ht_sync or in stream order.  ht_tracker_config clears every stream's debug
 * canvas; ht_tracker_set_params does not.
 * No two streams' outputs may share bytes: the streams of one tick run concurrently and would race, where the
 * reference's timers write one after another.
 * Errors (nothing changes): HT_ERR_STATE before ht_tracker_config; HT_ERR_ARG for a range outside [0, max_frames),
 * n <= 0, canvases NULL, a host pointer, a pointer or pitch that is not a multiple of 4, a pitch below 4*width, or a
 * canvas that overlaps any debug canvas, crop plane, tensor plane, camera, framed box or best-shot image or state of any stream after the call (the one
 * rule of ht_tracker_set_face_tensor); HT_ERR_SIZE for a size outside 1..16384. */
int ht_tracker_set_debug(ht_ctx *ctx, int first, int n, const ht_debug_canvas *canvases);

/* Stream first+i strokes main.js's face rectangles onto its debug canvas (enable[i] == 1) or not (0), for i in
 * [0, n).  After each tick, on top of that tick's back-projection, the library draws what src/main.js:199-219 strokes
 * for the tick's ht_tracker_event: a "VJ" record with confidence != 0 strokes its box in #0000CC, a "CS" record with
 * confidence != 0 its box rotated by angle - pi/2 about (x, y) in #00CC00 (a NaN angle: unrotated); other ticks draw
 * nothing.  The raster is the one of DESIGN.md 2, "Strokes": lineWidth 1, miter joins, butt caps, 16 x 16 samples
 * per pixel, non-premultiplied source-over, clipped to the canvas.  A stroke is a function of the record alone.
 * The flag belongs to the stream: ht_tracker_set_debug keeps it (a stream without a canvas draws nothing),
 * ht_tracker_config clears every stream's, ht_tracker_set_params, stop, start, reset and ht_tracker_import keep it.
 * While no stream has both the flag and a canvas, a tick launches nothing for strokes.
 * Errors (nothing changes): HT_ERR_STATE before ht_tracker_config; HT_ERR_ARG for a range outside [0, max_frames),
 * n <= 0, enable NULL, or a value other than 0 and 1. */
int ht_tracker_set_debug_strokes(ht_ctx *ctx, int first, int n, const int32_t *enable);

/* A stream's face crop: the tracked face cut out of its video, upright and at video resolution (DESIGN.md 2, "Face
 * crops").  Byte offsets: 0 rgba, 8 width, 12 height, 16 pitch, 20 pad_, 24 scale. */
typedef struct {
  uint8_t *rgba;          /* DEVICE memory, `height` rows of `pitch` bytes of RGBA8; NULL: the stream has no crop */
  int32_t width, height;  /* S_w x S_h, 1..2048 */
  int32_t pitch;          /* 0 -> 4*width; a multiple of 4, >= 4*width */
  int32_t pad_;
  double scale;           /* the face box is scaled by this about its centre; finite, in (0, 16] */
} ht_face_crop;           /* 32 bytes */
/* Stream first+i gets crops[i] (host array), for i in [0, n); stream states are kept.  After every tick whose record
 * is "CS" with width > 0 and height > 0 - track() kept the face - every pixel of the crop is written: the rectangle
 * main.js strokes in green (translate(x, y) . rotate(angle - pi/2), local box [ToInt32(-w/2), +w] x [ToInt32(-h/2),
 * +h]), scaled about its centre by `scale`, its shorter side grown until the aspect ratio is width : height, sampled
 * bilinearly from the tick's video (the frame ht_tracker_step was given, or the video of the feed record, through its
 * view) with 8-bit weights.  Taps outside the video or the view's source rectangle read (0, 0, 0, 0), so alpha shows
 * where the crop leaves the video.  Every other tick (IDLE, STARTING, WB, VJ - also the VJ tick that finds the face -
 * and the CS tick that loses it) leaves the crop as it was.  ht_face_crop_map gives the exact map.  The writes are
 * enqueued on the context's stream after the tick's records are computed: with host `out` they have landed when the
 * tick returns, with device `out` after ht_sync or in stream order.  The crop belongs to the stream id: stop, start,
 * reset, a lost face, ht_tracker_set_params and ht_tracker_import keep it; ht_tracker_config removes every stream's.
 * A tick launches one more kernel while some stream has a crop, and nothing more otherwise.
 * Errors (nothing changes): HT_ERR_STATE before ht_tracker_config; HT_ERR_ARG for a range outside [0, max_frames),
 * n <= 0, crops NULL, a host pointer, a pointer or pitch that is not a multiple of 4, a pitch below 4*width, a scale
 * that is not finite or outside (0, 16], or a crop that overlaps any debug canvas, crop plane, tensor plane, camera,
 * framed box or best-shot image or state of any stream after the call (the one rule of ht_tracker_set_face_tensor); HT_ERR_SIZE for a size outside 1..2048. */
int ht_tracker_set_face_crop(ht_ctx *ctx, int first, int n, const ht_face_crop *crops);

/* A stream's face crop as 4:2:0 video for an encoder: NVENC takes NV12; openh264, libx264, libvpx and WebRTC frame
 * buffers take I420 (DESIGN.md 2, "Face crops", item 5).  It is, bit for bit, the RGBA8 crop of the same size and
 * scale (ht_face_crop) converted with alpha ignored - so the part that leaves the video is black - by the library's one
 * RGB-to-YUV conversion: Y = y0 + ((yr R + yg G + yb B + 128) >> 8) per pixel, and per 2 x 2 block
 * U = clamp255(128 + ((ur SR + ug SG + ub SB + 512) >> 10)) of the block's sums (V likewise):
 *     color          y0   yr  yg  yb    ur   ug   ub    vr   vg   vb
 *     BT601          16   66 129  25   -38  -74  112   112  -94  -18
 *     BT709          16   47 157  16   -26  -86  112   112 -102  -10
 *     BT601 | FULL    0   77 150  29   -43  -85  128   128 -107  -21
 *     BT709 | FULL    0   54 183  19   -29  -99  128   128 -116  -12
 * Byte offsets, mirroring ht_yuv_image:
 *     0  uint8_t *planes[3]   DEVICE memory: NV12 Y, UV (U first), NULL; I420 Y, U, V; planes[0] NULL: no crop
 *    24  int32 pitch[3]       bytes per row; 0 -> tight (w, then w for NV12's UV or w/2 for I420's U and V); otherwise
 *                             >= that; any pointer or pitch alignment
 *    36  int32 width, height  S_w x S_h, both even, 2..2048
 *    44  int32 format         HT_YUV_NV12 or HT_YUV_I420
 *    48  int32 color          HT_YUV_BT601 or HT_YUV_BT709, optionally | HT_YUV_FULL_RANGE
 *    52  int32 pad_           0
 *    56  double scale         as ht_face_crop's */
typedef struct {
  uint8_t *planes[3];
  int32_t pitch[3];
  int32_t width, height;
  int32_t format;
  int32_t color;
  int32_t pad_;
  double scale;
} ht_face_crop_yuv;       /* 64 bytes */
/* Stream first+i gets the YUV crop crops[i] (host array), for i in [0, n).  A stream has at most one face crop in one
 * layout: this call and ht_tracker_set_face_crop each replace it, whatever its layout, and a NULL crop removes it.  It
 * is written on exactly the ticks, and lives exactly as long, as an RGBA crop (ht_tracker_set_face_crop); a tick with
 * crops of either layout launches one kernel more, and ht_face_crop_map gives its map (that of the RGBA crop of its
 * size and scale).
 * Errors (nothing changes; the message names the record): HT_ERR_STATE before ht_tracker_config; HT_ERR_SIZE for a size
 * that is odd or outside 2..2048; HT_ERR_ARG for a range outside [0, max_frames), n <= 0, crops NULL, a format other
 * than NV12 / I420, a colour other than the four above, a missing or extra plane, a host pointer, a pitch below its
 * row's bytes, a non-zero pad_, a scale that is not finite or outside (0, 16], or a plane that overlaps any debug
 * canvas, crop plane (its own crop's other planes included), tensor plane, camera, framed box or best-shot image or state of any stream after the call (the
 * one rule of ht_tracker_set_face_tensor). */
int ht_tracker_set_face_crop_yuv(ht_ctx *ctx, int first, int n, const ht_face_crop_yuv *crops);

/* A stream's face tensor: its face as a model's input, a normalised CHW or HWC tensor (DESIGN.md 2, "Face crops", item
 * 6).  It is a second output of the stream, next to and independent of its face crop.  It is, bit for bit, the RGBA8
 * crop of the same size and scale (ht_face_crop) with alpha ignored, converted per pixel P(i, j) = (R, G, B):
 *   channels  HT_TENSOR_RGB: c = R, G, B; HT_TENSOR_BGR: c = B, G, R; HT_TENSOR_GRAY: one channel,
 *             c = the detector's gray, ccv.grayscale: R 0.3 + G 0.59 + B 0.11 in fp64, left to right, stored
 *             round-half-even as a Uint8ClampedArray stores it
 *   value     HT_TENSOR_F32: v = fmaf((float)c, mul[k], add[k]), one rounding; HT_TENSOR_F16 / HT_TENSOR_BF16: that v
 *             rounded to nearest even (overflow gives +-inf); HT_TENSOR_U8: c itself (mul 1, add 0)
 *   layout    element (k, j, i) at data + k plane_stride + j row_stride + i (HT_TENSOR_CHW) or
 *             data + j row_stride + i C + k (HT_TENSOR_HWC), strides in elements; no other element is written
 * A pixel outside the video converts from (0, 0, 0): value add[k].  For a torchvision-style (x / 255 - mean) / std,
 * mul = 1 / (255 std) and add = -mean / std, each rounded once to float. */
#define HT_TENSOR_U8 0
#define HT_TENSOR_F16 1
#define HT_TENSOR_BF16 2
#define HT_TENSOR_F32 3
#define HT_TENSOR_CHW 0
#define HT_TENSOR_HWC 1
#define HT_TENSOR_RGB 0
#define HT_TENSOR_BGR 1
#define HT_TENSOR_GRAY 2
typedef struct {
  void *data;             /*  0 DEVICE memory of the context's device, aligned to the element size; NULL: none */
  int64_t row_stride;     /*  8 elements; CHW >= S_w, HWC >= C*S_w; at most 2^40 */
  int64_t plane_stride;   /* 16 elements; CHW with 3 channels: >= (S_h-1)*row_stride + S_w, at most 2^40; otherwise 0 */
  int32_t width, height;  /* 24 S_w x S_h, 1..2048 */
  int32_t dtype;          /* 32 HT_TENSOR_U8 / F16 / BF16 / F32 */
  int32_t layout;         /* 36 HT_TENSOR_CHW / HWC */
  int32_t channels;       /* 40 HT_TENSOR_RGB / BGR / GRAY */
  int32_t pad_;           /* 44 0 */
  float mul[3], add[3];   /* 48, 60 finite; GRAY uses [0]; U8: 1 and 0 */
  double scale;           /* 72 as ht_face_crop's, (0, 16] */
} ht_face_tensor;         /* 80 bytes */
/* Stream first+i gets the face tensor tensors[i] (host array), for i in [0, n); a NULL data removes the stream's.  A
 * stream has at most one tensor, and it is independent of the stream's face crop: ht_tracker_set_face_crop(_yuv) never
 * touch it, and this call never touches the crop.  It is written on exactly the ticks, and lives exactly as long, as a
 * crop: after every "CS" tick with width > 0 and height > 0, every element above is written; every other tick leaves
 * it as it was.  ht_face_crop_map gives its map (that of the RGBA crop of its size and scale).  The tensor belongs to
 * the stream id: stop, start, reset, a lost face, ht_tracker_set_params and ht_tracker_import keep it;
 * ht_tracker_config removes every stream's.  A tick with crops, tensors or both launches one kernel more, and nothing
 * more otherwise.  The tracker record format is unchanged.
 * Errors (nothing changes; the message names the record): HT_ERR_STATE before ht_tracker_config; HT_ERR_SIZE for a size
 * outside 1..2048; HT_ERR_ARG for a range outside [0, max_frames), n <= 0, tensors NULL, a dtype, layout or channels
 * value other than the above, a host pointer, a pointer not aligned to the element size, a stride outside its range
 * above, a non-zero pad_, a mul or add that is not finite, a U8 tensor whose used mul is not 1 or add not 0, a scale
 * that is not finite or outside (0, 16], or a tensor plane that overlaps any debug canvas, crop plane, tensor plane
 * (its own tensor's others included), camera, framed box or best-shot image or state of any stream after the call.
 * That is the one overlap rule of the per-stream outputs, which ht_tracker_set_debug, both crop setters and
 * ht_tracker_set_camera apply too: the streams of a tick run concurrently, so no two of the byte spans a tick writes
 * may share a byte.  The spans: each debug canvas, (height-1)*pitch + 4*width bytes; each plane of each face crop,
 * RGBA or YUV; each channel plane of a CHW tensor, or the whole of an HWC tensor; each camera, HT_CAMERA_BYTES; each
 * framed box (ht_tracker_set_framing), HT_FRAMED_BOX_BYTES; each best-shot image (ht_tracker_set_best_shot),
 * (height-1)*pitch + 4*width bytes, and each best-shot state, HT_BEST_SHOT_STATE_BYTES. */
int ht_tracker_set_face_tensor(ht_ctx *ctx, int first, int n, const ht_face_tensor *tensors);

/* The map of the crop `crop` (its size and scale; rgba and pitch are ignored; a YUV crop has the map of the RGBA crop of
 * its size and scale) for tracker record `ev`, on a canvas of
 * canvas_w x canvas_h drawn from a video_w x video_h video through `view` (NULL: the whole frame upright; for
 * ht_tracker_step the video is the canvas): crop pixel (i, j) samples video tap coordinates (U0 + i Ui + j Uj,
 * V0 + i Vi + j Vj) / 65536, with out = {U0, V0, Ui, Vi, Uj, Vj} exactly as the device computes them.  A tap coordinate
 * u is video pixel centre u + 1/2.  Host only; needs no context.  -> 1 if the record makes a crop, 0 if not (out all
 * 0), HT_ERR_ARG for NULL pointers, a scale outside (0, 16] or a bad view, HT_ERR_SIZE for a canvas or video outside
 * 1..16384 or a crop outside 1..2048. */
int ht_face_crop_map(const ht_tracker_event *ev, int canvas_w, int canvas_h, int video_w, int video_h,
                     const ht_video_view *view, const ht_face_crop *crop, int64_t out[6]);

/* A stream's framed box: the state of its framing (DESIGN.md 2, "Face crops", item 7), in caller-owned DEVICE memory,
 * an upright box in canvas pixels.  Byte offsets:
 *     0  double cx, cy            its centre
 *    16  double width, height     its size
 *    32  int32  canvas_w, canvas_h  the canvas it lies on
 *    40  uint32 updates           crop ticks applied since the framing was set
 *    44  int32  valid             0 until the first crop tick, then 1 */
typedef struct {
  double cx, cy;
  double width, height;
  int32_t canvas_w, canvas_h;
  uint32_t updates;
  int32_t valid;
} ht_framed_box;          /* 48 bytes */
#define HT_FRAMING_CROP 1     /* the face crop (RGBA or YUV) takes the framed box */
#define HT_FRAMING_TENSOR 2   /* the face tensor takes the framed box */
/* A stream's framing: a steady face-cam box that glides instead of jumping with every camshift box.  Explicit values:
 * the wrappers' defaults (alpha 0.25, dead zone 0.1) belong to the wrappers.  Byte offsets: 0 box, 8 alpha,
 * 16 dead_zone, 24 outputs, 28 pad_. */
typedef struct {
  ht_framed_box *box;     /* 8-byte aligned DEVICE memory of the context's device; NULL removes the framing */
  double alpha;           /* the share of the error outside the dead zone that a crop tick takes: (0, 1] */
  double dead_zone;       /* half-width of the dead zone, a fraction of the box's width (x) or height (y): [0, 0.5] */
  int32_t outputs;        /* HT_FRAMING_CROP | HT_FRAMING_TENSOR, nonzero: the outputs that take the framed box */
  int32_t pad_;           /* 0 */
} ht_framing;             /* 32 bytes */
/* Stream first+i gets framings[i] (host array), for i in [0, n); stream states are kept.  Setting a framing enqueues
 * its box to become invalid with updates = 0.  Then on every crop tick of the stream - a "CS" record with width > 0
 * and height > 0, the ticks that write face crops - the box moves, in fp64 with every operation rounded as written,
 * from its old state, towards the target: the centre (t_x, t_y) of the green rectangle as the crop places it, and the
 * record's width and height.  It snaps to the target when it is not valid, lies on another canvas size, or
 * |t_x - cx| > width / 2 or |t_y - cy| > height / 2 (the face has left the box); otherwise each of cx, cy, width,
 * height with target t moves by v += alpha (e - copysign(band, e)) where e = t - v exceeds band = dead_zone * the old
 * width (cx, width) or height (cy, height), and stays otherwise.  Every crop tick adds 1 to updates; other ticks leave
 * the box as it is.  The outputs named in `outputs` are then cut from the framed box instead of the record's: crop_map's
 * geometry with local centre (0, 0), no rotation and the box's centre and size, so they are always upright (with
 * alpha 1 and dead zone 0 an unrotated record gives exactly the tracked crop); the others keep the record's box.  Which
 * ticks write an output is unchanged.  The framing belongs to the stream id: stop, start, reset, a lost face,
 * ht_tracker_set_params and ht_tracker_import keep it; ht_tracker_config removes every stream's.  A tick launches one
 * more kernel while some stream has a framing, and nothing more otherwise.  ht_face_crop_map_framed gives the map.
 * Errors (nothing changes; the message names the record): HT_ERR_STATE before ht_tracker_config; HT_ERR_ARG for a
 * range outside [0, max_frames), n <= 0, framings NULL, a box that is host memory, memory of another device or not
 * 8-byte aligned, an alpha outside (0, 1] or a dead_zone outside [0, 0.5] (NaN included), an outputs mask that is 0
 * or has other bits, a non-zero pad_, or a box that overlaps any debug canvas, crop plane, tensor plane, camera or
 * framed box or best-shot image or state of any stream after the call (the one rule of ht_tracker_set_face_tensor; a box
 * is HT_FRAMED_BOX_BYTES). */
#define HT_FRAMED_BOX_BYTES 48
int ht_tracker_set_framing(ht_ctx *ctx, int first, int n, const ht_framing *framings);
/* The map of the crop `crop` (as for ht_face_crop_map) cut from framed box `box` (host memory) on a canvas_w x canvas_h
 * canvas drawn from a video_w x video_h video through `view`, exactly as the device computes it.  Host only.  -> 1, 0
 * for a box that is not valid (out all 0), or the errors of ht_face_crop_map. */
int ht_face_crop_map_framed(const ht_framed_box *box, int canvas_w, int canvas_h, int video_w, int video_h,
                            const ht_video_view *view, const ht_face_crop *crop, int64_t out[6]);

/* A stream's face redaction: its tracked face hidden in its own video, in place, after the tick's crops (DESIGN.md 2,
 * "Face redaction").  headtrackr tracks ONE face per stream: this hides the stream's tracked face, it is not a
 * detector of every face in the frame.  Explicit values: the wrappers' defaults (mosaic, block 16, scale 1.25, hold
 * 10, black) belong to the wrappers.  Byte offsets:
 *     0  int32  mode          HT_REDACT_OFF (removes the redaction), HT_REDACT_MOSAIC or HT_REDACT_FILL
 *     4  int32  block         B, the cell size in video pixels: even, 2..128
 *     8  int32  hold          0..65535 ticks the last face box stays redacted after the face is lost
 *    12  uint8  fill_rgb[3]   HT_REDACT_FILL on RGBA8 video and the packed RGB formats: R, G, B
 *    15  uint8  pad0          0
 *    16  uint8  fill_yuv[3]   HT_REDACT_FILL on the YUV formats: Y, U, V (8-bit; P010 writes v << 8)
 *    19  uint8  pad1          0
 *    20  int32  pad_          0
 *    24  double scale         the face box is scaled by this about its centre; finite, in (0, 16] */
#define HT_REDACT_OFF 0
#define HT_REDACT_MOSAIC 1
#define HT_REDACT_FILL 2
typedef struct {
  int32_t mode;
  int32_t block;
  int32_t hold;
  uint8_t fill_rgb[3];
  uint8_t pad0;
  uint8_t fill_yuv[3];
  uint8_t pad1;
  int32_t pad_;
  double scale;
} ht_face_redact;         /* 32 bytes */
/* Stream first+i gets redactions[i] (host array), for i in [0, n); stream states are kept, and the stream's hold
 * starts empty.  The library then WRITES the stream's video - the frames given to ht_tracker_step, the feed record's
 * planes - in place, although those pointers are const:
 *   face ticks   a record main.js strokes ("VJ" or "CS" with confidence != 0, the VJ tick that finds the face included,
 *                the CS tick that loses it not) with width, height > 0 and x, y, width, height finite and within 65536
 *   region       the VJ box upright, or the CS green rectangle as the face crop places it (angle - pi/2 about (x, y),
 *                a NaN angle unrotated), scaled by `scale` about its centre, its corners in fp64 scaled by sw / cw and
 *                sh / ch into the view's sw x sh source rectangle (the video without a view, the canvas for
 *                ht_tracker_step); pixels floor(min) .. ceil(max) - 1, clipped to the rectangle, through the view
 *   cells        every cell of a B x B grid anchored at video pixel (0, 0) that meets that, clipped to the rectangle
 *   values       in each channel a cell covers samples [x0 >> sx, ((x1 - 1) >> sx) + 1) (likewise in y), which become
 *                their integer mean (sum + cnt / 2) / cnt (mosaic; P010 on whole 16-bit words) or the fill; nothing
 *                else is written: no alpha, no pitch padding, no other pixel
 *   hold         a face tick stores its box and canvas size and sets remaining = hold; a later tick that ran a pass
 *                (detection != 0) on the same canvas size redacts that box through its own view and video while
 *                remaining > 0, taking one from it.  An IDLE tick, a canvas-size change or setting the redaction
 *                again ends the hold.
 * It runs last in the tick, after the face crops, tensors and the camshift model have read the unredacted video.  The
 * redaction belongs to the stream id: stop, start, reset, a lost face, ht_tracker_set_params and ht_tracker_import keep
 * it; ht_tracker_config removes every stream's.  A tick launches one more kernel while some stream has a redaction,
 * and nothing more otherwise.  It writes no caller buffer of its own, so the overlap rule of the outputs is unchanged.
 * Two rules then hold for every tick (ht_tracker_step and every feed), checked before anything is enqueued, with the
 * record named: a redacting stream's video must be device memory (a staged copy would hide the result), and no two
 * redacting records of one tick may have video planes that share a byte (their cells would race): one camera frame
 * shared through views may be redacted by one stream only.  Streams without a redaction are not affected.
 * Errors (nothing changes; the message names the record): HT_ERR_STATE before ht_tracker_config; HT_ERR_ARG for a
 * range outside [0, max_frames), n <= 0, redactions NULL, a mode other than the three, a block that is odd or outside
 * 2..128, a hold outside 0..65535, a non-zero pad, or a scale that is not finite or outside (0, 16]. */
int ht_tracker_set_redact(ht_ctx *ctx, int first, int n, const ht_face_redact *redactions);
/* The video rectangle a redaction `redact` (mode ignored) hides for face record `ev` on a canvas_w x canvas_h canvas
 * drawn from a video_w x video_h video through `view` (NULL: the whole frame upright), exactly as the device computes
 * it: video pixels [out[0], out[2]) x [out[1], out[3]), aligned to the B grid and clipped to the source rectangle.
 * Host only; needs no context.  -> 1, 0 for a record that is not a face tick or an empty region (out all 0),
 * HT_ERR_ARG for NULL pointers or a bad redaction or view, HT_ERR_SIZE for a canvas or video outside 1..16384. */
int ht_face_redact_rect(const ht_tracker_event *ev, int canvas_w, int canvas_h, int video_w, int video_h,
                        const ht_video_view *view, const ht_face_redact *redact, int32_t out[4]);

/* A stream's best shot: the sharpest face of its current or last track, one RGBA8 image per track (DESIGN.md 2, "Best
 * shots").  The state lives in caller-owned DEVICE memory.  Byte offsets:
 *     0  uint64 best_score     the score of the track's best tick
 *     8  uint64 score          the score of the stream's latest crop tick
 *    16  double x, y, width, height, angle   the best tick's record fields
 *    56  double now_ms         the best tick's clock
 *    64  int32  canvas_w, canvas_h   the best tick's canvas size (with x .. angle: ht_face_crop_map's input)
 *    72  uint32 track          tracks begun since the best shot was set; the current or last one is track
 *    76  uint32 ended          tracks ended; track t is final once ended >= t, a track is open while ended != track
 *    80  uint32 ticks          crop ticks in the current or last track
 *    84  uint32 best_tick      the best tick's index in that track, 0 for its first tick
 *    88  int32  buffer         the image the current or last track writes: rgba[buffer]
 *    92  uint32 flags          HT_BEST_* of the stream's latest tick (0: none of them) */
typedef struct {
  uint64_t best_score;
  uint64_t score;
  double x, y, width, height, angle;
  double now_ms;
  int32_t canvas_w, canvas_h;
  uint32_t track, ended;
  uint32_t ticks, best_tick;
  int32_t buffer;
  uint32_t flags;
} ht_best_shot_state;     /* 96 bytes */
#define HT_BEST_SHOT_STATE_BYTES 96
#define HT_BEST_BEGAN 1       /* the tick began a track */
#define HT_BEST_IMPROVED 2    /* the tick set the track's best (its first tick always does): rgba[buffer] was written */
#define HT_BEST_ENDED 4       /* the tick ended the open track (its best is final) */
/* A stream's best shot record.  Explicit values: the wrappers' default (scale 1) belongs to the wrappers.  Byte offsets:
 * 0 rgba[2], 16 state, 24 width, 28 height, 32 pitch, 36 pad_, 40 scale. */
typedef struct {
  uint8_t *rgba[2];       /* 4-byte aligned DEVICE images of S_h rows; rgba[0] NULL removes the best shot, rgba[1] NULL:
                             one image */
  ht_best_shot_state *state;  /* 8-byte aligned DEVICE memory of the context's device */
  int32_t width, height;  /* S_w x S_h, 3..2048 */
  int32_t pitch;          /* bytes per image row (both images); 0 = 4*width; a multiple of 4, >= 4*width */
  int32_t pad_;           /* 0 */
  double scale;           /* as ht_face_crop's, (0, 16] */
} ht_best_shot;           /* 48 bytes */
/* Stream first+i gets shots[i] (host array), for i in [0, n); stream states are kept.  Setting a best shot enqueues
 * its state to be zeroed (no track open); the images are not touched.  Then on every tick of the stream:
 *   crop tick   a "CS" record with width > 0 and height > 0 (the ticks that write face crops).  The candidate is, bit
 *               for bit, the RGBA8 face crop of the best shot's width, height and scale (ht_face_crop) from the tick's
 *               video, before any redaction; a framing never applies to it.  Its score is sum L^2 (uint64) over the
 *               pixels 1 <= i <= S_w-2, 1 <= j <= S_h-2 whose alpha and whose four neighbours' alphas are all 255, with
 *               L = 4 g(i,j) - g(i-1,j) - g(i+1,j) - g(i,j-1) - g(i,j+1) and g the detector's gray (HT_TENSOR_GRAY's).
 *               With no track open the tick begins track t = track + 1 (HT_BEST_BEGAN), whose image is rgba[(t-1) & 1]
 *               with two images and rgba[0] with one.  The track's first tick, and a later one whose score is strictly
 *               greater than best_score, set the best (HT_BEST_IMPROVED): the candidate is written to the image, every
 *               pixel, and the state takes its score and record.  The earliest tick wins a tie.
 *   other tick  (the CS tick that loses the face, any tick after stop or reset, ...) ends an open track (HT_BEST_ENDED).
 * ht_tracker_import ends the open tracks of the streams it writes (flags HT_BEST_ENDED): an imported stream is another
 * tracker.  A stream that a feed does not list does not tick: its track neither advances nor ends.  With two images
 * the previous track's final best stays intact for the whole next track.  The best shot belongs to the stream id:
 * stop, start, reset, ht_tracker_set_params and ht_tracker_import keep it; ht_tracker_config removes every stream's.  A
 * tick launches two more kernels while some stream has a best shot, and nothing more otherwise.  The tracker record
 * format is unchanged.
 * Errors (nothing changes; the message names the record): HT_ERR_STATE before ht_tracker_config; HT_ERR_SIZE for a size
 * outside 3..2048; HT_ERR_ARG for a range outside [0, max_frames), n <= 0, shots NULL, an image that is host memory or
 * not 4-byte aligned, a state that is host memory, memory of another device or not 8-byte aligned, a pitch that is not
 * a multiple of 4 >= 4*width, a non-zero pad_, a scale that is not finite or outside (0, 16], or an image or state that
 * overlaps any debug canvas, crop plane, tensor plane, camera, framed box, best-shot image (the shot's other image
 * included) or best-shot state of any stream after the call (the one rule of ht_tracker_set_face_tensor; an image is
 * (height-1)*pitch + 4*width bytes, a state HT_BEST_SHOT_STATE_BYTES). */
int ht_tracker_set_best_shot(ht_ctx *ctx, int first, int n, const ht_best_shot *shots);
/* The best-shot score of a w x h RGBA8 image (host memory, rows of `pitch` bytes, 0: 4*w), exactly as the device
 * computes it for a candidate.  Host only; needs no context.  -> HT_OK, HT_ERR_ARG for NULL pointers or a pitch below
 * 4*w, HT_ERR_SIZE for a size outside 3..2048. */
int ht_best_shot_score(const uint8_t *rgba, int w, int h, int pitch, uint64_t *out);

/* A stream's head-coupled camera: the three.js r48 PerspectiveCamera that realisticAbsoluteCameraControl moves
 * (src/controllers.js:28-68), in caller-owned DEVICE memory that a renderer can bind directly.  Byte offsets:
 *     0  double position[3]      camera.position
 *    24  double fov              camera.fov (degrees)
 *    32  double view[6]          setViewOffset(fullWidth, fullHeight, x, y, width, height); zeros before the first event
 *    80  uint32 events           headtrackingEvents applied since the controller was constructed
 *    84  int32  has_view_offset  0 until the first event, then 1
 *    88  float  projection[16]   projection matrix, column-major (DESIGN.md 5.4 f10)
 *   152  float  view_matrix[16]  inverse of the camera's world matrix T(position) R, column-major
 *   216  uint32 pad_[2]          0 */
typedef struct {
  double position[3];
  double fov;
  double view[6];
  uint32_t events;
  int32_t has_view_offset;
  float projection[16];
  float view_matrix[16];
  uint32_t pad_[2];
} ht_camera;
#define HT_CAMERA_BYTES 224
/* One stream's realisticAbsoluteCameraControl(camera, scaling, fixedPosition, lookAt, {screenHeight, damping}) and
 * the camera's own fov, aspect, near and far.  Explicit values: the reference's defaults (screenHeight 20, damping 1)
 * belong to the wrappers. */
typedef struct {
  ht_camera *camera;          /* 16-byte aligned DEVICE memory of the context's device; NULL removes the controller */
  double scaling;
  double fixed_position[3];
  double look_at[3];
  double screen_height, damping;
  double fov, aspect, near, far;
} ht_camera_control;          /* 112 bytes */
/* Stream first+i gets controls[i] (host array), for i in [0, n); stream states are kept.  Setting a controller
 * constructs it (src/controllers.js:40-46): the camera is enqueued to become position = fixed_position, fov = fov, no
 * view offset, events = 0, with the matrices of that state; R of the view matrix is fixed here by lookAt(fixed_position
 * -> look_at, up = +y), as the controller never calls lookAt again.  Setting one again re-constructs it.
 * Then on every tick whose record has head.valid - the reference dispatched a headtrackingEvent - the listener body
 * (src/controllers.js:48-67) runs on the device in fp64, in JavaScript's evaluation order, followed by
 * updateProjectionMatrix.  Ticks without one leave the camera as it is; the controller survives stop, start, reset and
 * a lost face, and ht_tracker_import (it is a device resource of the stream id, not part of the Tracker's state).  Each
 * stream hears only its own events.  The writes are enqueued on the context's stream after the tick's records are
 * computed: with host `out` they have landed when the tick returns, with device `out` after ht_sync or in stream order.
 * ht_tracker_config removes every controller; ht_tracker_set_params does not.  A tick launches one more kernel while
 * some stream has a controller, and nothing more otherwise.
 * Errors (nothing changes): HT_ERR_STATE before ht_tracker_config; HT_ERR_ARG for a range outside [0, max_frames),
 * n <= 0, controls NULL, a camera that is host memory, memory of another device or not 16-byte aligned, a camera that
 * overlaps any debug canvas, crop plane, tensor plane, camera, framed box or best-shot image or state of any stream after the call (the one rule of
 * ht_tracker_set_face_tensor), a non-finite field, aspect <= 0, near <= 0, far <= near, fov outside (0, 180), or a
 * degenerate lookAt (fixed_position == look_at, or a view direction parallel to +y). */
int ht_tracker_set_camera(ht_ctx *ctx, int first, int n, const ht_camera_control *controls);

/* Tracker records: a stream's whole headtrackr.Tracker as one fixed-size, position-independent, little-endian byte
 * string without pointers, so that a stream can move to another id, context or GPU, be cloned, or outlive its process.
 * Layout (byte offsets; the gaps between sections are zero):
 *       0  u32 magic HT_TRACKER_RECORD_MAGIC ("HTR1"), u32 format version HT_TRACKER_RECORD_VERSION,
 *          u32 record size HT_TRACKER_RECORD_BYTES, u32 0
 *      16  u64 checksum = sum of w_i * (2i + 1) mod 2^64 over the u32 words w_0, w_1, ... from byte 24 to the end
 *      32  the lifecycle state (280 bytes): mode, whitebalance window, "hints" timer, faceFound, Smoother, head
 *          diagonals, fov estimate, headposition state
 *     320  the stream's parameters as the device holds them (88 bytes, with the head-model constants)
 *     416  camshift section: the tracker (48 bytes: search window, TrackObj, angle, calcAngles, initialised),
 *     464  its two scheduling-history words (a pass count and window pixels / 256 of its last track()),
 *     480  its 4096-bin model histogram (u32)
 * Canonical form: when the stream's mode is not CS the camshift section is dead state (the next hand-off re-seeds it)
 * and is exported as zeros; so exporting an imported record gives the same bytes, and two exports of one state are
 * identical whatever the slot held before. */
#define HT_TRACKER_RECORD_BYTES 16864
#define HT_TRACKER_RECORD_MAGIC 0x31525448u
#define HT_TRACKER_RECORD_VERSION 1u
/* records[i] (HT_TRACKER_RECORD_BYTES each, contiguous) := stream streams[i], for i in [0, n).  One launch.
 *   streams: HOST array of n distinct ids in [0, max_frames), 1 <= n <= max_frames.
 *   records: host memory (returns after the records have landed) or 16-byte aligned device memory of the context's
 *            device (enqueue only: use ht_sync, or stream order on the context's stream).
 * Errors (nothing is enqueued): HT_ERR_STATE before ht_tracker_config; HT_ERR_ARG for n out of range, NULL pointers,
 * a device `streams`, an id out of range or listed twice, or device records of another device or misaligned. */
int ht_tracker_export(ht_ctx *ctx, const int32_t *streams, int n, void *records);
/* Stream streams[i] := records[i], for i in [0, n): its lifecycle state, parameters and camshift tracker become exactly
 * the exported stream's, and what it held before is discarded.  Its debug canvas (ht_tracker_set_debug), camera
 * controller (ht_tracker_set_camera) and framing with its box (ht_tracker_set_framing) stay as they were: those are
 * device resources of this stream id, not part of the
 * Tracker's state.  streams and records as for
 * ht_tracker_export; the source and the destination may be one context (clone: import into an idle id; swap: export
 * [a, b], import [b, a]).  Every record is checked on the device first - magic, format version (records of another
 * version are rejected, not converted), size, checksum, and every field that indexes an array or selects a branch:
 * mode in [0, 4], whitebalance samples in [0, 15], head diagonals in [0, 6], the parameters ht_tracker_set_params
 * accepts, and for a CS stream an initialised camshift tracker with a positive window - and the call synchronises.
 * Any failure is HT_ERR_ARG naming the first bad record in ht_last_error, and no stream changes.  On success the call
 * returns after the records have been consumed (also device records).  Two launches, whatever n. */
int ht_tracker_import(ht_ctx *ctx, const int32_t *streams, int n, const void *records);

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
 * the frames of call s must stay unchanged until then as well.  Consecutive pipelined calls may differ in frame size,
 * batch size and interval: the bin planes of the two calls in flight are the two fixed halves of one buffer, sized
 * for the largest max_frames x w x h pipelined so far (it grows only behind a synchronisation). */
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
