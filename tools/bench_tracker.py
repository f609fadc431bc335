#!/usr/bin/env python
"""Per-frame device time of ht_tracker_step (headtrackr.Tracker lifecycle) against ht_stream_step_head on the same
streams: N 640x480 streams, device-resident frames and outputs, CUDA events around each step.

  tracker_wb      ht_tracker_step while every stream is in the whitebalance gate
  tracker_cs      ht_tracker_step in steady tracking (every stream in "CS")
  stream_head_cs  ht_stream_step_head in steady tracking
  feed_*          ht_tracker_feed against ht_ingest + ht_tracker_step and ht_tracker_step (feed_arms)
  canvases_*      ht_tracker_feed_canvases on four canvas sizes against four one-size ht_tracker_feed calls, and
                  one-size ht_tracker_feed against another build of the library (--before-lib) (canvas_arms)
  migrate_*       (--migrate) ht_tracker_export + ht_tracker_import of every stream, device to device and through
                  pinned host memory, and a steady tick before and after an import (migrate_arms)
  strokes_*       (--strokes) ht_tracker_feed with a debug canvas on every stream and main.js's strokes on none,
                  1/64 and all of them, k_debug_strokes's kernel time, and the strokes-off arm against --before-lib
                  (strokes_arms)
  debug_*         (--debug-streams) ht_tracker_feed with debug canvases on none, 1/64 and all of the streams, the
                  achieved bandwidth of k_debug_backproj, and the no-debug arm against --before-lib (debug_arms)
  camera_*        (--camera-streams) ht_tracker_feed with head-coupled camera controllers on none, 1/64 and all of
                  the streams, k_camera_update's kernel time, and the no-controller arm against --before-lib
                  (camera_arms)
  yuv_* twopass_* rgba_*
                  (--yuv) ht_tracker_feed_yuv from NV12 video against ht_ingest_yuv + ht_tracker_feed and against
                  ht_tracker_feed from RGBA video of the same size (also --before-lib), and the draw kernels' time
                  (yuv_arms)
  <fmt>_*         (--formats) ht_tracker_feed_yuv from every video format against ht_ingest_yuv + ht_tracker_feed and
                  ht_tracker_feed from the converted RGBA video, NV12 / I420 / RGBA also against --before-lib, and
                  k_feed_draw_yuv's time per format (formats_arms)
  <fmt>_<config>_*
                  (--views) ht_tracker_feed(_yuv)_views from RGBA and NV12 video through rotations, mirrors and crops
                  against the plain feed of the upright video and against a separate rotate / crop pass + plain feed
                  (also --before-lib), and k_feed_draw_view's time (views_arms)
  crop*_* twopass*_*
                  (--crops) ht_tracker_feed_yuv from 1280x720 NV12 onto 320x240 canvases with 112x112 and 224x224 face
                  crops on none, 1/64 and all of the streams, against ht_ingest_yuv + grid_sample of the boxes (also
                  --before-lib), NV12 and I420 crops against RGBA crops + a torch conversion, and k_face_crop's time
                  (crops_arms)
  framing*_*      (--framing) the --crops workload with 224x224 NV12 crops on every stream, with a framing on no, every
                  and every 64th stream (no framing also against --before-lib), arms alternating tick by tick
                  (framing_arms)
  redact*_*       (--redact) 1024 streams of 1280x720 NV12 onto 320x240 canvases with a mosaic (B = 16, scale 1.5) on
                  no, every and every 64th stream (no redaction also against --before-lib), arms alternating tick by
                  tick, each arm on its own copy of the video (redact_arms)
  best*_*         (--best-shot) the --crops workload with 224x224 NV12 crops on every stream, with a 224x224 best
                  shot (two images) on no, every and every 64th stream (none also against --before-lib), arms
                  alternating tick by tick, and the kernel times of k_best_score and k_best_write (best_shot_arms)

Prints one JSON line with the card's name and power limit read in the same run; --out also writes it to a file."""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
        return name, power
    except Exception as e:  # the number is reported without them rather than not at all
        return f"unknown ({e})", "unknown"


def timed(torch, fn, steps):
    ts = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), float(min(ts))


def feed_arms(torch, frames, stream, N, W, H, steps, rounds):
    """ht_tracker_feed against the ways to get the same ticks without it, in steady tracking, every arm on its own
    context and all arms alternating tick by tick (the arm order rotates), CUDA events around each call:

      feed_cs          N streams, W x H device video drawn onto a W/2 x H/2 canvas by ht_tracker_feed
      ingest_step_cs   the same ticks as ht_ingest of the batch into a W/2 x H/2 canvas batch + ht_tracker_step
      feed_half_idle   feed_cs with every other stream stopped but still listed
      feed_1to1_cs     ht_tracker_feed of the W x H video onto a W x H canvas (the copy into the canvas arena) ...
      step_1to1_cs     ... against ht_tracker_step reading the same frames in place

    The records of the timed ticks must agree: feed_cs == ingest_step_cs, feed_1to1_cs == step_1to1_cs, and the running
    half of feed_half_idle == the same streams of feed_cs.  -> {arm_ms: median, arm_spread_ms: max - min of the
    per-round medians, ...}"""
    import ctypes as C
    from headtrackr_b200 import Context, _lib
    CW, CH = W // 2, H // 2
    rec_bytes = C.sizeof(_lib.TrackerEvent)
    now = [1.0e12]

    def records(n, w, h):
        arr = (_lib.VideoFrame * n)()
        for k in range(n):
            arr[k] = _lib.VideoFrame(frames[k].data_ptr(), k, w, h, 0, 0.0)
        return arr

    def feed_arm(cw, ch):
        c = Context(max_width=cw, max_height=ch, max_frames=N, stream=stream)
        arr, out = records(N, W, H), torch.empty(N * rec_bytes, dtype=torch.uint8, device="cuda")

        def prep():
            for k in range(N):
                arr[k].now_ms = now[0]

        def run():
            c._check(c._L.ht_tracker_feed(c._h, C.addressof(arr), N, 1, cw, ch, out.data_ptr()))
        return c, prep, run, out

    def ingest_step_arm():
        c = Context(max_width=CW, max_height=CH, max_frames=N, stream=stream)
        canvas = torch.empty((N, CH, CW, 4), dtype=torch.uint8, device="cuda")
        out = torch.empty(N * rec_bytes, dtype=torch.uint8, device="cuda")

        def run():
            c._check(c._L.ht_ingest(c._h, frames.data_ptr(), N, W, H, canvas.data_ptr(), CW, CH))
            c._check(c._L.ht_tracker_step(c._h, canvas.data_ptr(), N, CW, CH, now[0], out.data_ptr()))
        return c, None, run, out

    def step_arm():
        c = Context(max_width=W, max_height=H, max_frames=N, stream=stream)
        out = torch.empty(N * rec_bytes, dtype=torch.uint8, device="cuda")

        def run():
            c._check(c._L.ht_tracker_step(c._h, frames.data_ptr(), N, W, H, now[0], out.data_ptr()))
        return c, None, run, out

    arms = {"feed_cs": feed_arm(CW, CH), "ingest_step_cs": ingest_step_arm(), "feed_half_idle": feed_arm(CW, CH),
            "feed_1to1_cs": feed_arm(W, H), "step_1to1_cs": step_arm()}
    names = list(arms)
    for c, _, _, _ in arms.values():
        c.tracker_config()
        c.tracker_reset(0, N)
        c.tracker_start(0, N)

    def tick(name):
        c, prep, run, out = arms[name]
        if prep:
            prep()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        run()
        b.record()
        b.synchronize()
        return a.elapsed_time(b)

    def recs(name):
        return np.frombuffer(arms[name][3].cpu().numpy().tobytes(), np.uint8).reshape(N, rec_bytes)

    for _ in range(17):                          # the whitebalance gate, detection, the first CS frames
        now[0] += 20.0
        for name in names:
            tick(name)
    hc = arms["feed_half_idle"][0]
    for k in range(1, N, 2):                     # stop() every other stream; they stay listed
        hc.tracker_stop(k, 1)
    hc.sync()
    times = {name: [[] for _ in range(rounds)] for name in names}
    mismatches = 0
    for r in range(rounds):
        for s in range(steps):
            now[0] += 20.0
            rot = (r * steps + s) % len(names)
            for name in names[rot:] + names[:rot]:
                times[name][r].append(tick(name))
            fa, fb = recs("feed_cs"), recs("ingest_step_cs")
            mismatches += int((fa != fb).any(axis=1).sum())
            mismatches += int((recs("feed_1to1_cs") != recs("step_1to1_cs")).any(axis=1).sum())
            mismatches += int((recs("feed_half_idle")[0::2] != fa[0::2]).any(axis=1).sum())
    if mismatches:
        raise SystemExit(f"feed arms disagree on {mismatches} records of the timed ticks")
    res = {}
    for name in names:
        med = [float(np.median(t)) for t in times[name]]
        res[f"{name}_ms"] = float(np.median(sum(times[name], [])))
        res[f"{name}_spread_ms"] = max(med) - min(med)
    ev = [_lib.TrackerEvent.from_buffer_copy(bytes(row)) for row in recs("feed_cs")]
    res["feed_cs_streams"] = sum(e.detection == 2 for e in ev)
    ev = [_lib.TrackerEvent.from_buffer_copy(bytes(row)) for row in recs("feed_half_idle")]
    res["feed_half_idle_running"] = sum(e.running for e in ev)
    res["feed_canvas"] = f"{CW}x{CH}"
    res["feed_records_agree"] = True
    for c, _, _, _ in arms.values():
        c.close()
    return res


CANVASES = ((320, 240), (256, 192), (200, 150), (160, 120))


def other_build_context(before_lib, **kw):
    """a Context on another build of the library (e.g. the parent commit's).  It may predate entry points that
    _lib.lib() binds: bind only what the feed arms call."""
    import ctypes as C
    from headtrackr_b200 import Context, _lib
    L = C.CDLL(str(Path(before_lib).resolve()))
    vp = C.c_void_p
    L.ht_create.argtypes = [C.POINTER(vp), C.POINTER(_lib.Config), C.c_char_p, C.c_size_t]
    L.ht_destroy.argtypes, L.ht_destroy.restype = [vp], None
    L.ht_last_error.argtypes, L.ht_last_error.restype = [vp], C.c_char_p
    for f in (L.ht_sync, L.ht_max_rects):
        f.argtypes = [vp]
    L.ht_tracker_config.argtypes = [vp, vp]
    for f in (L.ht_tracker_reset, L.ht_tracker_start, L.ht_tracker_stop):
        f.argtypes = [vp, C.c_int, C.c_int]
    L.ht_tracker_feed.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp]
    if hasattr(L, "ht_tracker_feed_yuv"):
        L.ht_tracker_feed_yuv.argtypes = [vp, vp, C.c_int, C.c_int, vp]
    if hasattr(L, "ht_tracker_set_debug"):
        L.ht_tracker_set_debug.argtypes = [vp, C.c_int, C.c_int, vp]
    saved = _lib.lib
    _lib.lib = lambda: L
    try:
        return Context(**kw)
    finally:
        _lib.lib = saved


def canvas_arms(torch, frames, stream, N, W, H, steps, rounds, before_lib=None):
    """Streams with their own canvas sizes, in steady tracking; every arm on its own context, all arms alternating tick
    by tick (the arm order rotates), CUDA events around each tick:

      canvases_mixed_cs   N streams of W x H device video, stream k on canvas CANVASES[k % 4], in ONE
                          ht_tracker_feed_canvases call (four canvas-size groups: detection and camshift once per size)
      canvases_split_cs   the same ticks as four ht_tracker_feed calls, one per canvas size
      one_size_cs         ht_tracker_feed of all N streams onto CANVASES[0] (this build)
      one_size_before_cs  the same with the library at `before_lib` (another build, e.g. the parent commit's)

    The records must agree: mixed == split, one_size == one_size_before.  -> {arm_ms, arm_spread_ms, ...}"""
    import ctypes as C
    from headtrackr_b200 import Context, _lib
    rec_bytes = C.sizeof(_lib.TrackerEvent)
    MW, MH = max(c[0] for c in CANVASES), max(c[1] for c in CANVASES)
    now = [1.0e12]
    groups = [list(range(g, N, len(CANVASES))) for g in range(len(CANVASES))]

    def context():
        return Context(max_width=MW, max_height=MH, max_frames=N, stream=stream)

    def before_context():
        return other_build_context(before_lib, max_width=MW, max_height=MH, max_frames=N, stream=stream)

    def mixed_arm():
        c = context()
        arr = (_lib.CanvasFrame * N)()
        for k in range(N):
            cw, ch = CANVASES[k % len(CANVASES)]
            arr[k] = _lib.CanvasFrame(_lib.VideoFrame(frames[k].data_ptr(), k, W, H, 0, 0.0), cw, ch)
        out = torch.empty(N * rec_bytes, dtype=torch.uint8, device="cuda")

        def run():
            for k in range(N):
                arr[k].video.now_ms = now[0]
            c._check(c._L.ht_tracker_feed_canvases(c._h, C.addressof(arr), N, 1, out.data_ptr()))
        return c, run, out

    def split_arm():
        c = context()
        arrs = []
        for ks in groups:
            arr = (_lib.VideoFrame * len(ks))()
            for i, k in enumerate(ks):
                arr[i] = _lib.VideoFrame(frames[k].data_ptr(), k, W, H, 0, 0.0)
            arrs.append(arr)
        out = torch.empty(N * rec_bytes, dtype=torch.uint8, device="cuda")
        order = torch.tensor(sum(groups, []), device="cuda")
        inv = torch.empty_like(order)
        inv[order] = torch.arange(N, device="cuda")
        view = out.view(N, rec_bytes)

        def run():
            off = 0
            for (cw, ch), arr in zip(CANVASES, arrs):
                for i in range(len(arr)):
                    arr[i].now_ms = now[0]
                c._check(c._L.ht_tracker_feed(c._h, C.addressof(arr), len(arr), 1, cw, ch, view[off].data_ptr()))
                off += len(arr)
        return c, run, out, inv

    def one_size_arm(c):
        arr = (_lib.VideoFrame * N)()
        for k in range(N):
            arr[k] = _lib.VideoFrame(frames[k].data_ptr(), k, W, H, 0, 0.0)
        out = torch.empty(N * rec_bytes, dtype=torch.uint8, device="cuda")
        cw, ch = CANVASES[0]

        def run():
            for k in range(N):
                arr[k].now_ms = now[0]
            c._check(c._L.ht_tracker_feed(c._h, C.addressof(arr), N, 1, cw, ch, out.data_ptr()))
        return c, run, out

    mixed, split = mixed_arm(), split_arm()
    arms = {"canvases_mixed_cs": mixed[:3], "canvases_split_cs": split[:3], "one_size_cs": one_size_arm(context())}
    if before_lib:
        arms["one_size_before_cs"] = one_size_arm(before_context())
    names = list(arms)
    for c, _, _ in arms.values():
        c.tracker_config()
        c.tracker_reset(0, N)
        c.tracker_start(0, N)

    def tick(name):
        _, run, _ = arms[name]
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        run()
        b.record()
        b.synchronize()
        return a.elapsed_time(b)

    def recs(name):
        return arms[name][2].view(N, rec_bytes)

    for _ in range(17):                          # the whitebalance gate, detection, the first CS frames
        now[0] += 20.0
        for name in names:
            tick(name)
    times = {name: [[] for _ in range(rounds)] for name in names}
    mismatches = 0
    for r in range(rounds):
        for s in range(steps):
            now[0] += 20.0
            rot = (r * steps + s) % len(names)
            for name in names[rot:] + names[:rot]:
                times[name][r].append(tick(name))
            mismatches += int((recs("canvases_mixed_cs") != recs("canvases_split_cs")[split[3]]).any(dim=1).sum())
            if before_lib:
                mismatches += int((recs("one_size_cs") != recs("one_size_before_cs")).any(dim=1).sum())
    if mismatches:
        raise SystemExit(f"canvas arms disagree on {mismatches} records of the timed ticks")
    res = {}
    for name in names:
        med = [float(np.median(t)) for t in times[name]]
        res[f"{name}_ms"] = float(np.median(sum(times[name], [])))
        res[f"{name}_spread_ms"] = max(med) - min(med)
    ev = [_lib.TrackerEvent.from_buffer_copy(bytes(row)) for row in recs("canvases_mixed_cs").cpu().numpy()]
    res["canvases_mixed_cs_streams"] = sum(e.detection == 2 for e in ev)
    ev = [_lib.TrackerEvent.from_buffer_copy(bytes(row)) for row in recs("one_size_cs").cpu().numpy()]
    res["one_size_cs_streams"] = sum(e.detection == 2 for e in ev)
    res["canvases"] = ["%dx%d" % c for c in CANVASES]
    res["canvas_records_agree"] = True
    for c, _, _ in arms.values():
        c.close()
    return res


HBM_BYTES_PER_S = 3.35e12       # H100 SXM HBM3, NVIDIA data sheet


def debug_arms(torch, frames, stream, N, W, H, steps, rounds, before_lib=None):
    """Debug canvases (ht_tracker_set_debug) in steady tracking: N streams of W x H device video fed onto W x H canvases
    by ht_tracker_feed, every arm on its own context, all arms alternating tick by tick (the arm order rotates), CUDA
    events around each tick:

      debug0_cs         no stream has a debug canvas (the tick launches what it launched before debug canvases)
      debug64_cs        every 64th stream has a W x H debug canvas
      debugall_cs       every stream has one
      debug0_before_cs  debug0_cs with the library at `before_lib` (e.g. the parent commit's build)

    Then, in a run of its own under torch.profiler, the kernel time of k_debug_table and k_debug_backproj over `steps`
    ticks of debugall_cs, and k_debug_backproj's achieved bytes/s: per CS entry with a canvas it reads the 2-byte bin
    plane (2*w*h) and writes the clipped image (4*min(w,Dw)*min(h,Dh)); k_debug_table reads the model and current
    histograms (2 * 16 KB) and writes a 4112-byte table.  The records of every arm must agree."""
    import ctypes as C
    from headtrackr_b200 import Context, _lib
    rec_bytes = C.sizeof(_lib.TrackerEvent)
    now = [1.0e12]
    recs_arr = (_lib.VideoFrame * N)()
    for k in range(N):
        recs_arr[k] = _lib.VideoFrame(frames[k].data_ptr(), k, W, H, 0, 0.0)
    kw = dict(max_width=W, max_height=H, max_frames=N, stream=stream)
    canvases = {}

    def arm(every, before=False):
        c = other_build_context(before_lib, **kw) if before else Context(**kw)
        c.tracker_config()
        c.tracker_reset(0, N)
        c.tracker_start(0, N)
        if every:
            dbg = [torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda") if k % every == 0 else None for k in range(N)]
            c.tracker_set_debug(0, dbg)
            canvases[every] = sum(d is not None for d in dbg)
        return c, torch.empty(N * rec_bytes, dtype=torch.uint8, device="cuda")

    arms = {"debug0_cs": arm(0), "debug64_cs": arm(64), "debugall_cs": arm(1)}
    if before_lib:
        arms["debug0_before_cs"] = arm(0, before=True)
    names = list(arms)

    def tick(name):
        c, out = arms[name]
        for k in range(N):
            recs_arr[k].now_ms = now[0]
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        c._check(c._L.ht_tracker_feed(c._h, C.addressof(recs_arr), N, 1, W, H, out.data_ptr()))
        b.record()
        b.synchronize()
        return a.elapsed_time(b)

    for _ in range(17):                          # the whitebalance gate, detection, the first CS frames
        now[0] += 20.0
        for name in names:
            tick(name)
    times = {name: [[] for _ in range(rounds)] for name in names}
    for r in range(rounds):
        for s in range(steps):
            now[0] += 20.0
            rot = (r * steps + s) % len(names)
            for name in names[rot:] + names[:rot]:
                times[name][r].append(tick(name))
            first = arms[names[0]][1].cpu()
            if any(not torch.equal(first, arms[name][1].cpu()) for name in names[1:]):
                raise SystemExit("debug arms disagree on the records of a timed tick")
    res = {}
    for name in names:
        med = [float(np.median(t)) for t in times[name]]
        res[f"{name}_ms"] = float(np.median(sum(times[name], [])))
        res[f"{name}_spread_ms"] = max(med) - min(med)
    ev = [_lib.TrackerEvent.from_buffer_copy(bytes(row))
          for row in arms["debugall_cs"][1].cpu().numpy().reshape(N, rec_bytes)]
    cs = sum(e.detection == 2 for e in ev)
    res["debug_cs_streams"] = cs
    res["debug64_canvases"], res["debugall_canvases"] = canvases[64], canvases[1]
    res["debug_records_agree"] = True

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            now[0] += 20.0
            tick("debugall_cs")
        torch.cuda.synchronize()
    kernel_us = {}
    for e in prof.key_averages():
        for kname in ("k_debug_backproj", "k_debug_table"):
            if kname in e.key:
                t = getattr(e, "device_time_total", None)
                kernel_us[kname] = kernel_us.get(kname, 0.0) + (t if t is not None else e.cuda_time_total)
    for kname, us in kernel_us.items():
        res[f"{kname}_ms"] = us / 1000.0 / steps
    bp_bytes = cs * (2 * W * H + 4 * W * H)
    tab_bytes = cs * (2 * 4 * 4096 + 4112)
    res["k_debug_backproj_bytes"] = bp_bytes
    if "k_debug_backproj" in kernel_us:
        rate = bp_bytes / (kernel_us["k_debug_backproj"] / steps * 1e-6)
        res["k_debug_backproj_TBps"] = rate / 1e12
        res["k_debug_backproj_of_3.35TBps"] = rate / HBM_BYTES_PER_S
    if "k_debug_table" in kernel_us:
        res["k_debug_table_GBps"] = tab_bytes / (kernel_us["k_debug_table"] / steps * 1e-6) / 1e9
    for c, _ in arms.values():
        c.close()
    return res


def strokes_arms(torch, frames, stream, N, W, H, steps, rounds, before_lib=None):
    """Strokes (ht_tracker_set_debug_strokes) in steady tracking: N streams of W x H device video fed onto W x H canvases
    by ht_tracker_feed, every stream with a W x H debug canvas, every arm on its own context, all arms alternating
    tick by tick (the arm order rotates), CUDA events around each tick:

      strokes0_cs         no stream strokes (the tick launches what it launched before strokes)
      strokes64_cs        every 64th stream strokes
      strokesall_cs       every stream strokes
      strokes0_before_cs  strokes0_cs with the library at `before_lib` (e.g. the parent commit's build)

    Then, in a run of its own under torch.profiler, the kernel time of k_debug_strokes over `steps` ticks of
    strokesall_cs.  The records of every arm must agree."""
    import ctypes as C
    from headtrackr_b200 import Context, _lib
    rec_bytes = C.sizeof(_lib.TrackerEvent)
    now = [1.0e12]
    recs_arr = (_lib.VideoFrame * N)()
    for k in range(N):
        recs_arr[k] = _lib.VideoFrame(frames[k].data_ptr(), k, W, H, 0, 0.0)
    kw = dict(max_width=W, max_height=H, max_frames=N, stream=stream)

    def arm(every, before=False):
        c = other_build_context(before_lib, **kw) if before else Context(**kw)
        c.tracker_config()
        c.tracker_reset(0, N)
        c.tracker_start(0, N)
        c.tracker_set_debug(0, [torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda") for _ in range(N)])
        if every:
            c.tracker_set_debug_strokes(0, [k % every == 0 for k in range(N)])
        return c, torch.empty(N * rec_bytes, dtype=torch.uint8, device="cuda")

    arms = {"strokes0_cs": arm(0), "strokes64_cs": arm(64), "strokesall_cs": arm(1)}
    if before_lib:
        arms["strokes0_before_cs"] = arm(0, before=True)
    names = list(arms)

    def tick(name):
        c, out = arms[name]
        for k in range(N):
            recs_arr[k].now_ms = now[0]
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        c._check(c._L.ht_tracker_feed(c._h, C.addressof(recs_arr), N, 1, W, H, out.data_ptr()))
        b.record()
        b.synchronize()
        return a.elapsed_time(b)

    for _ in range(17):                          # the whitebalance gate, detection, the first CS frames
        now[0] += 20.0
        for name in names:
            tick(name)
    times = {name: [[] for _ in range(rounds)] for name in names}
    for r in range(rounds):
        for s in range(steps):
            now[0] += 20.0
            rot = (r * steps + s) % len(names)
            for name in names[rot:] + names[:rot]:
                times[name][r].append(tick(name))
            first = arms[names[0]][1].cpu()
            if any(not torch.equal(first, arms[name][1].cpu()) for name in names[1:]):
                raise SystemExit("stroke arms disagree on the records of a timed tick")
    res = {}
    for name in names:
        med = [float(np.median(t)) for t in times[name]]
        res[f"{name}_ms"] = float(np.median(sum(times[name], [])))
        res[f"{name}_spread_ms"] = max(med) - min(med)
    ev = [_lib.TrackerEvent.from_buffer_copy(bytes(row))
          for row in arms["strokesall_cs"][1].cpu().numpy().reshape(N, rec_bytes)]
    res["strokes_cs_streams"] = sum(e.detection == 2 for e in ev)
    res["strokes_records_agree"] = True

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            now[0] += 20.0
            tick("strokesall_cs")
        torch.cuda.synchronize()
    us = 0.0
    for e in prof.key_averages():
        if "k_debug_strokes" in e.key:
            t = getattr(e, "device_time_total", None)
            us += t if t is not None else e.cuda_time_total
    res["k_debug_strokes_ms"] = us / 1000.0 / steps
    for c, _ in arms.values():
        c.close()
    return res


def camera_arms(torch, frames, stream, N, W, H, steps, rounds, before_lib=None):
    """Camera controllers (ht_tracker_set_camera) in steady tracking with head positions: N streams of W x H device
    video fed onto W x H canvases by ht_tracker_feed, every arm on its own context, all arms alternating tick by tick
    (the arm order rotates), CUDA events around each tick:

      camera0_cs         no stream has a controller (the tick launches what it launched before controllers)
      camera64_cs        every 64th stream has one
      cameraall_cs       every stream has one
      camera0_before_cs  camera0_cs with the library at `before_lib` (e.g. the parent commit's build)

    Then, in a run of its own under torch.profiler, the kernel time of k_camera_update over `steps` ticks of
    cameraall_cs.  The records of every arm must agree."""
    import ctypes as C
    from headtrackr_b200 import Context, _lib
    rec_bytes = C.sizeof(_lib.TrackerEvent)
    now = [1.0e12]
    recs_arr = (_lib.VideoFrame * N)()
    for k in range(N):
        recs_arr[k] = _lib.VideoFrame(frames[k].data_ptr(), k, W, H, 0, 0.0)
    kw = dict(max_width=W, max_height=H, max_frames=N, stream=stream)
    cams, counts = {}, {}
    control = dict(scaling=1.0, fixedPosition=[0.0, 0.0, 0.0], lookAt=[0.0, 0.0, -1.0], fov=75.0, aspect=4 / 3,
                   near=1.0, far=10000.0)

    def arm(every, before=False):
        c = other_build_context(before_lib, **kw) if before else Context(**kw)
        c.tracker_config()
        c.tracker_reset(0, N)
        c.tracker_start(0, N)
        if every:
            buf = torch.zeros(N * _lib.CAMERA_BYTES, dtype=torch.uint8, device="cuda")
            c.tracker_set_camera(0, [dict(control, out=buf[_lib.CAMERA_BYTES * k: _lib.CAMERA_BYTES * (k + 1)])
                                     if k % every == 0 else None for k in range(N)])
            cams[every] = buf
            counts[every] = len(range(0, N, every))
        return c, torch.empty(N * rec_bytes, dtype=torch.uint8, device="cuda")

    arms = {"camera0_cs": arm(0), "camera64_cs": arm(64), "cameraall_cs": arm(1)}
    if before_lib:
        arms["camera0_before_cs"] = arm(0, before=True)
    names = list(arms)

    def tick(name):
        c, out = arms[name]
        for k in range(N):
            recs_arr[k].now_ms = now[0]
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        c._check(c._L.ht_tracker_feed(c._h, C.addressof(recs_arr), N, 1, W, H, out.data_ptr()))
        b.record()
        b.synchronize()
        return a.elapsed_time(b)

    for _ in range(30):                          # the whitebalance gate, detection, CS until the head diagonal is stable
        now[0] += 20.0
        for name in names:
            tick(name)
    times = {name: [[] for _ in range(rounds)] for name in names}
    for r in range(rounds):
        for s in range(steps):
            now[0] += 20.0
            rot = (r * steps + s) % len(names)
            for name in names[rot:] + names[:rot]:
                times[name][r].append(tick(name))
            first = arms[names[0]][1].cpu()
            if any(not torch.equal(first, arms[name][1].cpu()) for name in names[1:]):
                raise SystemExit("camera arms disagree on the records of a timed tick")
    res = {}
    for name in names:
        med = [float(np.median(t)) for t in times[name]]
        res[f"{name}_ms"] = float(np.median(sum(times[name], [])))
        res[f"{name}_spread_ms"] = max(med) - min(med)
    ev = [_lib.TrackerEvent.from_buffer_copy(bytes(row))
          for row in arms["cameraall_cs"][1].cpu().numpy().reshape(N, rec_bytes)]
    res["camera_head_events_per_tick"] = sum(e.head.valid for e in ev)
    res["camera64_controllers"], res["cameraall_controllers"] = counts[64], counts[1]
    res["camera_records_agree"] = True
    res["cameraall_events_min"] = min(int(v) for v in cams[1].view(N, _lib.CAMERA_BYTES)[:, 80:84].cpu().numpy()
                                      .view(np.uint32).ravel())

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            now[0] += 20.0
            tick("cameraall_cs")
        torch.cuda.synchronize()
    us = 0.0
    for e in prof.key_averages():
        if "k_camera_update" in e.key:
            t = getattr(e, "device_time_total", None)
            us += t if t is not None else e.cuda_time_total
    res["k_camera_update_ms"] = us / 1000.0 / steps
    for c, _ in arms.values():
        c.close()
    return res


YUV_LAYOUTS = [((1280, 720), (320, 240)), ((1280, 720), (640, 480)), ((640, 480), (640, 480))]


def nv12_streams(torch, N, W, H):
    """N NV12 device videos of W x H (BT.601 limited range) -> (Y planes (N, H, W), UV planes (N, H/2, W)).  Each
    stream its own video: one of 8 synth frames, shifted right by its own offset, so that every tick reads N distinct
    frames from HBM as N cameras would."""
    from headtrackr_b200 import synth
    base = torch.stack([torch.from_numpy(synth.frame(i, W, H, n_faces=1)) for i in range(8)]).cuda()
    ys = torch.empty((N, H, W), dtype=torch.uint8, device="cuda")
    uvs = torch.empty((N, H // 2, W), dtype=torch.uint8, device="cuda")
    for k0 in range(0, N, 64):
        k1 = min(N, k0 + 64)
        f = torch.stack([torch.roll(base[k % 8], shifts=2 * (k // 8) % 64, dims=1) for k in range(k0, k1)]).float()
        r, g, b = f[..., 0], f[..., 1], f[..., 2]
        y = 16 + (65.481 * r + 128.553 * g + 24.966 * b) / 255
        u = 128 + (-37.797 * r - 74.203 * g + 112.0 * b) / 255
        v = 128 + (112.0 * r - 93.786 * g - 18.214 * b) / 255
        uv = torch.stack([u[:, 0::2, 0::2], v[:, 0::2, 0::2]], dim=-1).reshape(k1 - k0, H // 2, W)
        ys[k0:k1] = torch.floor(y + 0.5).clamp(0, 255).to(torch.uint8)
        uvs[k0:k1] = torch.floor(uv + 0.5).clamp(0, 255).to(torch.uint8)
    return ys, uvs


def crop_theta(torch, ev, W, H, CW, CH, Sw, Sh, scale):
    """affine_grid thetas (N, 2, 3) of the face crops of device records `ev` (N x 144 bytes) in fp32: the geometry of
    DESIGN.md 2, "Face crops" as a caller writes it with torch (records without a crop give some finite theta)"""
    import math
    f = ev.view(torch.float64).reshape(ev.numel() // 144, 18)
    x, y, w, h, angle = (f[:, i].float() for i in (1, 2, 3, 4, 5))
    t = torch.nan_to_num(angle - math.pi / 2, nan=0.0)
    s, c = torch.sin(t), torch.cos(t)
    cx, cy = torch.trunc(-w / 2) + w / 2, torch.trunc(-h / 2) + h / 2
    hw, hh = w * scale / 2, h * scale / 2
    hw, hh = torch.maximum(hw, hh * Sw / Sh), torch.maximum(hh, hw * Sh / Sw)
    kx, ky = W / CW, H / CH
    # video coordinates of crop point (p, q): x = a p + b q + e, y = d p + g q + k (pixel centres at +0.5)
    a, b, d, g = c * 2 * hw / Sw * kx, -s * 2 * hh / Sh * kx, s * 2 * hw / Sw * ky, c * 2 * hh / Sh * ky
    lx, ly = cx - hw, cy - hh
    e, k = (x + c * lx - s * ly) * kx, (y + s * lx + c * ly) * ky
    # normalised output (u, v) in [-1, 1] is crop point ((u + 1) Sw / 2, (v + 1) Sh / 2); input x -> 2 x / W - 1
    row0 = torch.stack([a * Sw / W, b * Sh / W, (a * Sw / 2 + b * Sh / 2 + e) * 2 / W - 1], 1)
    row1 = torch.stack([d * Sw / H, g * Sh / H, (d * Sw / 2 + g * Sh / 2 + k) * 2 / H - 1], 1)
    return torch.stack([row0, row1], 1)


def torch_nv12(torch, rgba):
    """(N, S, S, 4) uint8 RGBA crops -> (Y (N, S, S), UV (N, S/2, S)) uint8: the library's BT.601 limited-range
    conversion (DESIGN.md 2, "Face crops", item 5) as a caller writes it in torch"""
    c = rgba[..., :3].to(torch.int32)
    r, g, b = c[..., 0], c[..., 1], c[..., 2]
    y = 16 + ((66 * r + 129 * g + 25 * b + 128) >> 8)
    s = c.reshape(c.shape[0], c.shape[1] // 2, 2, c.shape[2] // 2, 2, 3).sum(dim=(2, 4))
    sr, sg, sb = s[..., 0], s[..., 1], s[..., 2]
    u = (128 + ((-38 * sr - 74 * sg + 112 * sb + 512) >> 10)).clamp(0, 255)
    v = (128 + ((112 * sr - 94 * sg - 18 * sb + 512) >> 10)).clamp(0, 255)
    return y.to(torch.uint8), torch.stack([u, v], -1).reshape(c.shape[0], c.shape[1] // 2, c.shape[2]).to(torch.uint8)


def crops_arms(torch, stream, N, steps, rounds, before_lib=None):
    """Face crops (ht_tracker_set_face_crop) in steady tracking: N streams of 1280x720 NV12 device video fed onto
    320x240 canvases by ht_tracker_feed_yuv, every arm on its own context, all arms alternating tick by tick (the arm
    order rotates), CUDA events around each tick:

      crop0_cs              no crops (the tick launches what it launched before crops)
      crop0_before_cs       crop0_cs with the library at `before_lib` (e.g. the parent commit's build)
      crop<S>all_cs         an S x S crop (S = 112, 224) on every stream, scale 1
      crop<S>64_cs          an S x S crop on every 64th stream
      twopass<S>_cs         what a caller does without crops: the crops-off tick, ht_ingest_yuv of every video to
                            RGBA8 at video size, then torch's grid_sample (fp16, bilinear) of every stream's box
      crop<S>nv12_cs        an S x S NV12 crop on every stream (ht_tracker_set_face_crop_yuv, BT.601)
      crop<S>i420_cs        an S x S I420 crop on every stream
      rgbaconv<S>_cs        what a caller who encodes crops does without YUV crops: the crop<S>all tick, then the
                            same BT.601 conversion to NV12 written in torch (integer ops on the device)
      crop<S>all_before_cs  crop<S>all_cs with the library at `before_lib`
      tensor<S>_cs          an S x S fp16 CHW RGB face tensor on every stream, normalised with ImageNet's mean / std
                            (ht_tracker_set_face_tensor through Context.face_tensor_batch), no crop
      tensornv12<S>_cs      that tensor and an S x S NV12 crop on every stream (one k_face_crop, two grid slices)
      rgbanorm<S>_cs        what a caller who feeds a model does without tensors: the crop<S>all tick, then
                            crop[..., :3].permute(0, 3, 1, 2).float().div(255).sub(mean).div(std).half() into a batch

    Then, in runs of their own under torch.profiler, k_face_crop's kernel time per tick in the crop<S>all,
    crop<S>nv12 / crop<S>i420, tensor<S>, tensornv12<S> and crop<S>all_before arms.  The records of every arm must
    agree on every timed tick, every YUV crop must equal the torch conversion of the RGBA crop of its stream, and the
    largest difference between the tensors and the torch normalise pass is reported."""
    import ctypes as C
    import torch.nn.functional as F
    from headtrackr_b200 import Context, _lib
    from headtrackr_b200.context import _yuv_image
    W, H, CW, CH = 1280, 720, 320, 240
    rec_bytes = C.sizeof(_lib.TrackerEvent)
    now = [1.0e12]
    kw = dict(max_width=CW, max_height=CH, max_frames=N, stream=stream)
    ys, uvs = nv12_streams(torch, N, W, H)
    keep = []
    imgs = [_yuv_image((ys[k], uvs[k]), "nv12", "bt601", keep)[0] for k in range(N)]
    yrecs = (_lib.YuvFrame * N)()
    for k in range(N):
        yrecs[k] = _lib.YuvFrame(imgs[k], k, CW, CH, 0, 0.0)
    ingest_src = (_lib.YuvImage * N)(*imgs)
    rgba = torch.empty((N, H, W, 4), dtype=torch.uint8, device="cuda")
    crops = {S: torch.zeros((N, S, S, 4), dtype=torch.uint8, device="cuda") for S in (112, 224)}

    def planes(S, fmt):
        def z(h, w):
            return torch.zeros((N, h, w), dtype=torch.uint8, device="cuda")
        return (z(S, S), z(S // 2, S)) if fmt == "nv12" else (z(S, S), z(S // 2, S // 2), z(S // 2, S // 2))
    yuv = {(S, fmt): planes(S, fmt) for S in (112, 224) for fmt in ("nv12", "i420")}
    twopass_out, conv_out, norm_out, tens = {}, {}, {}, {}
    mean, std = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
    mean_t = torch.tensor(mean, device="cuda").view(1, 3, 1, 1)
    std_t = torch.tensor(std, device="cuda").view(1, 3, 1, 1)

    def arm(kind, S=0, every=0):
        c = other_build_context(before_lib, **kw) if kind == "before" else Context(**kw)
        c.tracker_config()
        c.tracker_reset(0, N)
        c.tracker_start(0, N)
        if kind in ("nv12", "i420", "tensornv12"):
            fmt = "nv12" if kind == "tensornv12" else kind
            c.tracker_set_face_crop(0, [{"out": tuple(p[k] for p in yuv[(S, fmt)]), "format": fmt, "color": "bt601"}
                                        for k in range(N)])
        elif every:
            c.tracker_set_face_crop(0, [{"out": crops[S][k]} if k % every == 0 else None for k in range(N)])
        if kind in ("tensor", "tensornv12"):
            tens[(S, kind)] = c.face_tensor_batch(0, N, S, S, torch.float16, "chw", "rgb", mean, std)
        out = torch.empty(N * rec_bytes, dtype=torch.uint8, device="cuda")

        def run():
            for k in range(N):
                yrecs[k].now_ms = now[0]
            c._check(c._L.ht_tracker_feed_yuv(c._h, C.addressof(yrecs), N, 1, out.data_ptr()))
            if kind == "twopass":
                c._check(c._L.ht_ingest_yuv(c._h, C.addressof(ingest_src), N, 1, rgba.data_ptr(), W, H))
                theta = crop_theta(torch, out, W, H, CW, CH, S, S, 1.0)
                src = rgba.permute(0, 3, 1, 2).half()
                grid = F.affine_grid(theta.half(), (N, 4, S, S), align_corners=False)
                twopass_out[S] = F.grid_sample(src, grid, mode="bilinear", padding_mode="zeros", align_corners=False)
            if kind == "rgbaconv":
                conv_out[S] = torch_nv12(torch, crops[S])
            if kind == "rgbanorm":
                norm_out[S] = crops[S][..., :3].permute(0, 3, 1, 2).float().div(255).sub(mean_t).div(std_t).half()
        return c, run, out

    arms = {"crop0_cs": arm("plain"), "crop112all_cs": arm("crop", 112, 1), "crop11264_cs": arm("crop", 112, 64),
            "crop224all_cs": arm("crop", 224, 1), "crop22464_cs": arm("crop", 224, 64),
            "twopass112_cs": arm("twopass", 112), "twopass224_cs": arm("twopass", 224)}
    for S in (112, 224):
        arms[f"crop{S}nv12_cs"], arms[f"crop{S}i420_cs"] = arm("nv12", S), arm("i420", S)
        arms[f"rgbaconv{S}_cs"] = arm("rgbaconv", S, 1)
        arms[f"tensor{S}_cs"], arms[f"tensornv12{S}_cs"] = arm("tensor", S), arm("tensornv12", S)
        arms[f"rgbanorm{S}_cs"] = arm("rgbanorm", S, 1)
    if before_lib:
        arms["crop0_before_cs"] = arm("before")
        for S in (112, 224):
            arms[f"crop{S}all_before_cs"] = arm("before", S, 1)
    names = list(arms)

    def tick(name):
        _, run, _ = arms[name]
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        run()
        b.record()
        b.synchronize()
        return a.elapsed_time(b)

    for _ in range(17):                          # the whitebalance gate, detection, the first CS frames
        now[0] += 20.0
        for name in names:
            tick(name)
    times = {name: [[] for _ in range(rounds)] for name in names}
    for r in range(rounds):
        for s in range(steps):
            now[0] += 20.0
            rot = (r * steps + s) % len(names)
            for name in names[rot:] + names[:rot]:
                times[name][r].append(tick(name))
            first = arms[names[0]][2]
            if any(not torch.equal(first, arms[name][2]) for name in names[1:]):
                raise SystemExit("crop arms disagree on the records of a timed tick")
    res = {}
    for name in names:
        med = [float(np.median(t)) for t in times[name]]
        res[f"{name}_ms"] = float(np.median(sum(times[name], [])))
        res[f"{name}_spread_ms"] = max(med) - min(med)
    ev = [_lib.TrackerEvent.from_buffer_copy(bytes(row)) for row in arms["crop0_cs"][2].cpu().numpy().reshape(N, rec_bytes)]
    cs = [e.detection == 2 and e.width > 0 and e.height > 0 for e in ev]
    res["crops_cs_streams"] = sum(cs)
    res["crops_records_agree"] = True
    for S in (112, 224):                         # the two paths cut the same faces (different resamplers)
        fused = crops[S].permute(0, 3, 1, 2).float()[torch.tensor(cs, device="cuda")]
        two = twopass_out[S].float()[torch.tensor(cs, device="cuda")]
        res[f"twopass{S}_vs_fused_mean_abs_diff"] = float((fused - two).abs().mean())
        # every YUV crop is the conversion of its RGBA crop (streams that never kept a face have no crop yet)
        m = torch.tensor(cs, device="cuda")
        want = torch_nv12(torch, crops[S])
        y, uv = yuv[(S, "nv12")]
        y4, u4, v4 = yuv[(S, "i420")]
        res[f"crop{S}_yuv_equals_converted_rgba"] = bool(
            torch.equal(y[m], want[0][m]) and torch.equal(uv[m], want[1][m]) and torch.equal(y4[m], want[0][m]) and
            torch.equal(u4[m], want[1][..., 0::2][m]) and torch.equal(v4[m], want[1][..., 1::2][m]) and
            torch.equal(conv_out[S][0], want[0]) and torch.equal(conv_out[S][1], want[1]))
        # the tensors against the torch normalise pass of the RGBA crops (one fmaf against two-step fp32, then fp16)
        res[f"tensor{S}_vs_torch_norm_max_abs_diff"] = max(
            float((tens[(S, kind)][m].float() - norm_out[S][m].float()).abs().max()) for kind in ("tensor", "tensornv12"))
        res[f"tensor{S}_equals_tensornv12"] = bool(torch.equal(tens[(S, "tensor")][m], tens[(S, "tensornv12")][m]))

    from torch.profiler import ProfilerActivity, profile
    for S in (112, 224):
        for layout, bpp in (("all", 4), ("nv12", 1.5), ("i420", 1.5), ("tensor", 6), ("tensornv12", 7.5)) + \
                ((("all_before", 4),) if before_lib else ()):
            arm_name = f"{layout}{S}_cs" if layout.startswith("tensor") else f"crop{S}{layout}_cs"
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(steps):
                    now[0] += 20.0
                    arms[arm_name][1]()
                torch.cuda.synchronize()
            us = 0.0
            for e in prof.key_averages():
                if "k_face_crop" in e.key:
                    t = getattr(e, "device_time_total", None)
                    us += t if t is not None else e.cuda_time_total
            name = f"k_face_crop_{S}" + ("" if layout == "all" else f"_{layout}")
            res[f"{name}_ms"] = us / 1000.0 / steps
            res[f"{name}_write_GBps"] = N * S * S * bpp / (us * 1e-6 / steps) / 1e9 if us > 0 else None
    for c, _, _ in arms.values():
        c.close()
    return res


def yuv_arms(torch, stream, N, steps, rounds, before_lib=None):
    """YUV video (ht_tracker_feed_yuv) in steady tracking, for each (video, canvas) of YUV_LAYOUTS: N streams, each
    with its own NV12 device video (BT.601 limited range), every arm on its own context, all arms of a layout
    alternating tick by tick (the arm order rotates), CUDA events around each tick:

      yuv_<layout>_cs          ht_tracker_feed_yuv from the NV12 planes onto the canvas
      twopass_<layout>_cs      ht_ingest_yuv of the batch into a device RGBA buffer of the video's size, then
                               ht_tracker_feed from it (what a caller writes without ht_tracker_feed_yuv)
      rgba_<layout>_cs         ht_tracker_feed from RGBA video of the same size (the converted frames)
      rgba_before_<layout>_cs  the same with the library at `before_lib` (e.g. the parent commit's build)

    Then, in runs of their own under torch.profiler, the kernel time of the draw per tick: k_feed_draw_yuv in the yuv
    arm, k_feed_draw in the rgba arm, with the bytes each must move (plane or RGBA bytes of the video read once, RGBA
    canvas written) over that time.  The records of every arm must agree on every timed tick."""
    import ctypes as C
    from headtrackr_b200 import Context, _lib, synth
    from headtrackr_b200.context import _yuv_image
    rec_bytes = C.sizeof(_lib.TrackerEvent)
    res = {}
    for (W, H), (CW, CH) in YUV_LAYOUTS:
        lay = f"{W}x{H}_{CW}x{CH}"
        now = [1.0e12]
        kw = dict(max_width=CW, max_height=CH, max_frames=N, stream=stream)
        ys, uvs = nv12_streams(torch, N, W, H)
        planes = [(ys[k], uvs[k]) for k in range(N)]
        keep = []
        imgs = [_yuv_image(p, "nv12", "bt601", keep)[0] for p in planes]
        conv = Context(max_width=CW, max_height=CH, max_frames=1, stream=stream)
        rgba = torch.empty((N, H, W, 4), dtype=torch.uint8, device="cuda")      # the converted video, for the RGBA arms
        conv.ingest_yuv(planes, W, H, out=rgba)
        conv.sync()
        conv.close()
        yrecs = (_lib.YuvFrame * N)()
        vrecs = (_lib.VideoFrame * N)()
        for k in range(N):
            yrecs[k] = _lib.YuvFrame(imgs[k], k, CW, CH, 0, 0.0)
            vrecs[k] = _lib.VideoFrame(rgba[k].data_ptr(), k, W, H, 0, 0.0)
        ingest_src = (_lib.YuvImage * N)(*imgs)
        staged = torch.empty((N, H, W, 4), dtype=torch.uint8, device="cuda")
        srecs = (_lib.VideoFrame * N)()
        for k in range(N):
            srecs[k] = _lib.VideoFrame(staged[k].data_ptr(), k, W, H, 0, 0.0)

        def arm(kind):
            c = other_build_context(before_lib, **kw) if kind == "rgba_before" else Context(**kw)
            c.tracker_config()
            c.tracker_reset(0, N)
            c.tracker_start(0, N)
            out = torch.empty(N * rec_bytes, dtype=torch.uint8, device="cuda")

            def run():
                t = now[0]
                if kind == "yuv":
                    for k in range(N):
                        yrecs[k].now_ms = t
                    c._check(c._L.ht_tracker_feed_yuv(c._h, C.addressof(yrecs), N, 1, out.data_ptr()))
                    return
                recs = vrecs
                if kind == "twopass":
                    c._check(c._L.ht_ingest_yuv(c._h, C.addressof(ingest_src), N, 1, staged.data_ptr(), W, H))
                    recs = srecs
                for k in range(N):
                    recs[k].now_ms = t
                c._check(c._L.ht_tracker_feed(c._h, C.addressof(recs), N, 1, CW, CH, out.data_ptr()))
            return c, run, out

        kinds = ["yuv", "twopass", "rgba"] + (["rgba_before"] if before_lib else [])
        arms = {k: arm(k) for k in kinds}

        def tick(name):
            _, run, _ = arms[name]
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            run()
            b.record()
            b.synchronize()
            return a.elapsed_time(b)

        for _ in range(17):                      # the whitebalance gate, detection, the first CS frames
            now[0] += 20.0
            for name in kinds:
                tick(name)
        times = {name: [[] for _ in range(rounds)] for name in kinds}
        for r in range(rounds):
            for s in range(steps):
                now[0] += 20.0
                rot = (r * steps + s) % len(kinds)
                for name in kinds[rot:] + kinds[:rot]:
                    times[name][r].append(tick(name))
                first = arms["yuv"][2]
                if any(not torch.equal(first, arms[name][2]) for name in kinds[1:]):
                    raise SystemExit(f"yuv arms disagree on the records of a timed tick ({lay})")
        for name in kinds:
            med = [float(np.median(t)) for t in times[name]]
            res[f"{name}_{lay}_cs_ms"] = float(np.median(sum(times[name], [])))
            res[f"{name}_{lay}_cs_spread_ms"] = max(med) - min(med)
        ev = [_lib.TrackerEvent.from_buffer_copy(bytes(row)) for row in arms["yuv"][2].cpu().numpy().reshape(N, rec_bytes)]
        res[f"yuv_{lay}_cs_streams"] = sum(e.detection == 2 for e in ev)

        from torch.profiler import ProfilerActivity, profile
        canvas_bytes = N * CW * CH * 4
        for name, kernel, video_bytes in (("yuv", "k_feed_draw_yuv", N * W * H * 3 // 2), ("rgba", "k_feed_draw", N * W * H * 4)):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(steps):
                    now[0] += 20.0
                    arms[name][1]()
                torch.cuda.synchronize()
            us = 0.0
            for e in prof.key_averages():
                base = e.key.split("(")[0].split("<")[0]
                if base.endswith(kernel) and (kernel == "k_feed_draw_yuv" or not base.endswith("k_feed_draw_yuv")):
                    t = getattr(e, "device_time_total", None)
                    us += t if t is not None else e.cuda_time_total
            ms = us / 1000.0 / steps
            res[f"{kernel}_{lay}_ms"] = ms
            res[f"{kernel}_{lay}_gb_per_s"] = (video_bytes + canvas_bytes) / (ms * 1e-3) / 1e9 if ms > 0 else None
        for c, _, _ in arms.values():
            c.close()
        del staged, rgba, planes, keep, ys, uvs
        torch.cuda.empty_cache()
    res["yuv_records_agree"] = True
    return res


FORMATS = ["nv21", "i422", "i444", "yuyv", "uyvy", "p010", "bgra", "bgr24", "rgb24", "nv12", "i420"]


def format_video(torch, rgba, fmt):
    """(N, H, W, 4) uint8 device RGBA -> the same video in `fmt` as Context takes it, one frame per stream (a test-local
    BT.601 limited-range RGB -> YUV, chroma from the block's first pixel; P010 with the 8-bit value in the top byte)"""
    N, H, W = rgba.shape[:3]
    if fmt in ("bgra", "bgr24", "rgb24"):
        order = {"bgra": [2, 1, 0, 3], "bgr24": [2, 1, 0], "rgb24": [0, 1, 2]}[fmt]
        v = rgba[..., order].contiguous()
        return [v[k] for k in range(N)]
    f = rgba.float()
    r, g, b = f[..., 0], f[..., 1], f[..., 2]
    q = lambda a: torch.floor(a + 0.5).clamp(0, 255).to(torch.uint8)     # noqa: E731
    y = q(16 + (65.481 * r + 128.553 * g + 24.966 * b) / 255)
    u = q(128 + (-37.797 * r - 74.203 * g + 112.0 * b) / 255)
    v = q(128 + (112.0 * r - 93.786 * g - 18.214 * b) / 255)
    del f, r, g, b
    if fmt == "i444":
        return [(y[k], u[k].contiguous(), v[k].contiguous()) for k in range(N)]
    if fmt in ("i422", "yuyv", "uyvy"):
        u2, v2 = u[:, :, 0::2].contiguous(), v[:, :, 0::2].contiguous()
        if fmt == "i422":
            return [(y[k], u2[k], v2[k]) for k in range(N)]
        a, c = (y[:, :, 0::2], u2) if fmt == "yuyv" else (u2, y[:, :, 0::2])
        bb, d = (y[:, :, 1::2], v2) if fmt == "yuyv" else (v2, y[:, :, 1::2])
        p = torch.stack([a, c, bb, d], dim=-1).reshape(N, H, W, 2)
        return [p[k] for k in range(N)]
    u4, v4 = u[:, 0::2, 0::2], v[:, 0::2, 0::2]
    if fmt == "i420":
        return [(y[k], u4[k].contiguous(), v4[k].contiguous()) for k in range(N)]
    pair = torch.stack([v4, u4] if fmt == "nv21" else [u4, v4], dim=-1).reshape(N, H // 2, W)
    if fmt == "p010":
        w16 = lambda a: (a.to(torch.int32) << 8).to(torch.int16)           # noqa: E731
        y16, p16 = w16(y), w16(pair)
        return [(y16[k], p16[k]) for k in range(N)]
    return [(y[k], pair[k]) for k in range(N)]


def formats_arms(torch, stream, N, steps, rounds, before_lib=None):
    """Every video format (ht_tracker_feed_yuv) in steady tracking, for each (video, canvas) of YUV_LAYOUTS: N streams,
    each with its own device video, every arm on its own context, the arms of a (layout, format) alternating tick by
    tick (the order rotates), CUDA events around each tick:

      <fmt>_<layout>_cs          ht_tracker_feed_yuv from the video in <fmt>
      <fmt>_twopass_<layout>_cs  ht_ingest_yuv of the batch into a device RGBA buffer, then ht_tracker_feed
      <fmt>_rgba_<layout>_cs     ht_tracker_feed from the RGBA frames the conversion makes
      <fmt>_before_<layout>_cs   (nv12, i420) ht_tracker_feed_yuv with the library at `before_lib`
      <fmt>_rgba_before_<layout>_cs  (nv12) the RGBA arm with the library at `before_lib`

    Then, in runs of their own under torch.profiler, k_feed_draw_yuv's time per tick for each format and its achieved
    bytes/s (video bytes read once + canvas written).  The records of every arm must agree on every timed tick."""
    import ctypes as C
    from headtrackr_b200 import Context, _lib, synth
    from headtrackr_b200.context import _yuv_image
    rec_bytes = C.sizeof(_lib.TrackerEvent)
    res = {}
    for (W, H), (CW, CH) in YUV_LAYOUTS:
        lay = f"{W}x{H}_{CW}x{CH}"
        kw = dict(max_width=CW, max_height=CH, max_frames=N, stream=stream)
        base = torch.stack([torch.from_numpy(synth.frame(i, W, H, n_faces=1)) for i in range(8)]).cuda()
        rgba = torch.empty((N, H, W, 4), dtype=torch.uint8, device="cuda")
        for k in range(N):
            rgba[k] = torch.roll(base[k % 8], shifts=2 * (k // 8) % 64, dims=1)
        del base
        conv = torch.empty_like(rgba)
        staged = torch.empty_like(rgba)
        for fmt in FORMATS:
            now = [1.0e12]
            vid = format_video(torch, rgba, fmt)
            keep = []
            imgs = [_yuv_image(v, fmt, "bt601", keep)[0] for v in vid]
            cc = Context(max_width=CW, max_height=CH, max_frames=1, stream=stream)
            cc.ingest_yuv(vid, W, H, fmt, out=conv)
            cc.sync()
            cc.close()
            yrecs = (_lib.YuvFrame * N)(*[_lib.YuvFrame(imgs[k], k, CW, CH, 0, 0.0) for k in range(N)])
            vrecs = (_lib.VideoFrame * N)(*[_lib.VideoFrame(conv[k].data_ptr(), k, W, H, 0, 0.0) for k in range(N)])
            srecs = (_lib.VideoFrame * N)(*[_lib.VideoFrame(staged[k].data_ptr(), k, W, H, 0, 0.0) for k in range(N)])
            ingest_src = (_lib.YuvImage * N)(*imgs)

            def arm(kind):
                before = kind.endswith("before")
                c = other_build_context(before_lib, **kw) if before else Context(**kw)
                c.tracker_config()
                c.tracker_reset(0, N)
                c.tracker_start(0, N)
                out = torch.empty(N * rec_bytes, dtype=torch.uint8, device="cuda")

                def run():
                    t = now[0]
                    if kind in ("fmt", "before"):
                        for k in range(N):
                            yrecs[k].now_ms = t
                        c._check(c._L.ht_tracker_feed_yuv(c._h, C.addressof(yrecs), N, 1, out.data_ptr()))
                        return
                    recs = vrecs
                    if kind == "twopass":
                        c._check(c._L.ht_ingest_yuv(c._h, C.addressof(ingest_src), N, 1, staged.data_ptr(), W, H))
                        recs = srecs
                    for k in range(N):
                        recs[k].now_ms = t
                    c._check(c._L.ht_tracker_feed(c._h, C.addressof(recs), N, 1, CW, CH, out.data_ptr()))
                return c, run, out

            kinds = ["fmt", "twopass", "rgba"]
            if before_lib and fmt in ("nv12", "i420"):
                kinds.append("before")
            if before_lib and fmt == "nv12":
                kinds.append("rgba_before")
            arms = {k: arm(k) for k in kinds}

            def tick(name):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                arms[name][1]()
                b.record()
                b.synchronize()
                return a.elapsed_time(b)

            for _ in range(17):
                now[0] += 20.0
                for name in kinds:
                    tick(name)
            times = {name: [[] for _ in range(rounds)] for name in kinds}
            for r in range(rounds):
                for s in range(steps):
                    now[0] += 20.0
                    rot = (r * steps + s) % len(kinds)
                    for name in kinds[rot:] + kinds[:rot]:
                        times[name][r].append(tick(name))
                    if any(not torch.equal(arms["fmt"][2], arms[name][2]) for name in kinds[1:]):
                        raise SystemExit(f"format arms disagree on the records of a timed tick ({fmt}, {lay})")
            for name in kinds:
                med = [float(np.median(t)) for t in times[name]]
                key = fmt if name == "fmt" else f"{fmt}_{name}"
                res[f"{key}_{lay}_cs_ms"] = float(np.median(sum(times[name], [])))
                res[f"{key}_{lay}_cs_spread_ms"] = max(med) - min(med)
            ev = [_lib.TrackerEvent.from_buffer_copy(bytes(row)) for row in arms["fmt"][2].cpu().numpy().reshape(N, rec_bytes)]
            res[f"{fmt}_{lay}_cs_streams"] = sum(e.detection == 2 for e in ev)

            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(steps):
                    now[0] += 20.0
                    arms["fmt"][1]()
                torch.cuda.synchronize()
            us = 0.0
            for e in prof.key_averages():
                if e.key.split("(")[0].split("<")[0].endswith("k_feed_draw_yuv"):
                    t = getattr(e, "device_time_total", None)
                    us += t if t is not None else e.cuda_time_total
            ms = us / 1000.0 / steps
            video_bytes = N * sum(t.numel() * t.element_size() for t in (vid[0] if isinstance(vid[0], tuple) else (vid[0],)))
            res[f"k_feed_draw_yuv_{fmt}_{lay}_ms"] = ms
            res[f"k_feed_draw_yuv_{fmt}_{lay}_tb_per_s"] = (video_bytes + N * CW * CH * 4) / (ms * 1e-3) / 1e12 if ms > 0 else None
            for c, _, _ in arms.values():
                c.close()
            del vid, keep, imgs
            torch.cuda.empty_cache()
        del rgba, conv, staged
        torch.cuda.empty_cache()
    res["formats_records_agree"] = True
    return res


# (name, video W x H, canvas, orientation, crop of the oriented frame or None)
VIEW_CONFIGS = [("identity", (1280, 720), (320, 240), 0, None), ("rot180", (1280, 720), (320, 240), 2, None),
                ("mirror", (1280, 720), (320, 240), 4, None), ("crop960", (1280, 720), (320, 240), 0, (160, 0, 960, 720)),
                ("rot90", (1280, 720), (240, 320), 1, None), ("rot270", (1280, 720), (240, 320), 3, None),
                ("1to1", (640, 480), (640, 480), 0, None), ("1to1_rot90", (640, 480), (480, 640), 1, None)]


def views_arms(torch, stream, N, steps, rounds, before_lib=None):
    """Video drawn through views (ht_tracker_feed_views / ht_tracker_feed_yuv_views) in steady tracking, RGBA and NV12,
    for each of VIEW_CONFIGS: N streams, each with its own device video V in memory orientation, every arm on its own
    context, the arms alternating tick by tick (the order rotates), CUDA events around each tick:

      <fmt>_<config>_view_cs     the feed of V through the view
      <fmt>_<config>_plain_cs    the plain feed (ht_tracker_feed / ht_tracker_feed_yuv) of the upright crop of V,
                                 prepared beforehand, on the same canvas
      <fmt>_<config>_twopass_cs  ht_ingest(_yuv)_views of V into an RGBA buffer of the crop's size, then ht_tracker_feed
      <fmt>_<config>_before_cs   the plain arm with the library at `before_lib` (e.g. the parent commit's build)

    Then, in a run of its own under torch.profiler, k_feed_draw_view's time per tick and its achieved bytes/s (video
    bytes read once + canvas written), and the plain arm's draw kernel.  The records of every arm must agree on every
    timed tick (even-sized 4:2:0 orientations and crops keep chroma blocks whole, so the upright NV12 twin is exact)."""
    import ctypes as C
    from headtrackr_b200 import Context, _lib, synth, views
    from headtrackr_b200.context import _views, _yuv_image
    rec_bytes = C.sizeof(_lib.TrackerEvent)
    res = {}

    def unorient(a, o):          # V with orient(V, o) == a, on the first two dimensions
        return torch.rot90(torch.flip(a, dims=(1,)) if o & 4 else a, o & 3, dims=(0, 1)).contiguous()

    for name, (W, H), (CW, CH), o, crop in VIEW_CONFIGS:
        OW, OH = (H, W) if o & 1 else (W, H)
        sx, sy, sw, sh = crop or (0, 0, OW, OH)
        v = {"rotate": 90 * (o & 3), "mirror": bool(o & 4), "crop": crop}
        assert views.oriented_size(v, W, H) == (OW, OH)
        base = torch.stack([torch.from_numpy(synth.frame(i, OW, OH, n_faces=1)) for i in range(8)]).cuda()
        up = torch.empty((N, OH, OW, 4), dtype=torch.uint8, device="cuda")     # the oriented frames O
        for k in range(N):
            up[k] = torch.roll(base[k % 8], shifts=2 * (k // 8) % 64, dims=1)
        del base
        for fmt in ("rgba", "nv12"):
            kw = dict(max_width=max(CW, 640), max_height=max(CH, 640), max_frames=N, stream=stream)
            keep = []
            if fmt == "rgba":
                vid = [unorient(up[k], o) for k in range(N)]
                plain = [up[k, sy:sy + sh, sx:sx + sw].contiguous() for k in range(N)]
                vrecs = [_lib.VideoFrame(x.data_ptr(), k, W, H, 0, 0.0) for k, x in enumerate(vid)]
                precs = (_lib.VideoFrame * N)(*[_lib.VideoFrame(x.data_ptr(), k, sw, sh, 0, 0.0) for k, x in enumerate(plain)])
                vcanv = (_lib.CanvasFrame * N)(*[_lib.CanvasFrame(r, CW, CH) for r in vrecs])
                ingest_src = (_lib.VideoFrame * N)(*vrecs)
            else:
                yu = format_video(torch, up, "nv12")                           # the oriented frames in NV12
                pair = lambda p: p.reshape(p.shape[0], p.shape[1] // 2, 2)      # noqa: E731
                vid = [(unorient(y, o), unorient(pair(uv), o).reshape(H // 2, W)) for y, uv in yu]
                plain = [(y[sy:sy + sh, sx:sx + sw].contiguous(), uv[sy // 2:(sy + sh) // 2, sx:sx + sw].contiguous())
                         for y, uv in yu]
                del yu
                imgs = [_yuv_image(x, "nv12", "bt601", keep)[0] for x in vid]
                pimgs = [_yuv_image(x, "nv12", "bt601", keep)[0] for x in plain]
                vcanv = (_lib.YuvFrame * N)(*[_lib.YuvFrame(imgs[k], k, CW, CH, 0, 0.0) for k in range(N)])
                precs = (_lib.YuvFrame * N)(*[_lib.YuvFrame(pimgs[k], k, CW, CH, 0, 0.0) for k in range(N)])
                ingest_src = (_lib.YuvImage * N)(*imgs)
            staged = torch.empty((N, sh, sw, 4), dtype=torch.uint8, device="cuda")
            srecs = (_lib.VideoFrame * N)(*[_lib.VideoFrame(staged[k].data_ptr(), k, sw, sh, 0, 0.0) for k in range(N)])
            vviews = _views(v, N)
            now = [1.0e12]

            def arm(kind):
                c = other_build_context(before_lib, **kw) if kind == "before" else Context(**kw)
                c.tracker_config()
                c.tracker_reset(0, N)
                c.tracker_start(0, N)
                out = torch.empty(N * rec_bytes, dtype=torch.uint8, device="cuda")

                def run():
                    t = now[0]
                    if kind == "view":
                        for k in range(N):
                            if fmt == "rgba":
                                vcanv[k].video.now_ms = t
                            else:
                                vcanv[k].now_ms = t
                        f = c._L.ht_tracker_feed_views if fmt == "rgba" else c._L.ht_tracker_feed_yuv_views
                        c._check(f(c._h, C.addressof(vcanv), C.addressof(vviews), N, 1, out.data_ptr()))
                        return
                    recs = precs
                    if kind == "twopass":
                        f = c._L.ht_ingest_views if fmt == "rgba" else c._L.ht_ingest_yuv_views
                        c._check(f(c._h, C.addressof(ingest_src), C.addressof(vviews), N, 1, staged.data_ptr(), sw, sh))
                        recs = srecs
                    for k in range(N):
                        recs[k].now_ms = t
                    if fmt == "nv12" and kind != "twopass":
                        c._check(c._L.ht_tracker_feed_yuv(c._h, C.addressof(recs), N, 1, out.data_ptr()))
                    else:
                        c._check(c._L.ht_tracker_feed(c._h, C.addressof(recs), N, 1, CW, CH, out.data_ptr()))
                return c, run, out

            kinds = ["view", "plain", "twopass"] + (["before"] if before_lib else [])
            arms = {k: arm(k) for k in kinds}

            def tick(arm_name):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                arms[arm_name][1]()
                b.record()
                b.synchronize()
                return a.elapsed_time(b)

            for _ in range(17):
                now[0] += 20.0
                for k in kinds:
                    tick(k)
            times = {k: [[] for _ in range(rounds)] for k in kinds}
            for r in range(rounds):
                for s in range(steps):
                    now[0] += 20.0
                    rot = (r * steps + s) % len(kinds)
                    for k in kinds[rot:] + kinds[:rot]:
                        times[k][r].append(tick(k))
                    if any(not torch.equal(arms["view"][2], arms[k][2]) for k in kinds[1:]):
                        raise SystemExit(f"view arms disagree on the records of a timed tick ({fmt}, {name})")
            key = f"{fmt}_{name}"
            for k in kinds:
                med = [float(np.median(t)) for t in times[k]]
                res[f"{key}_{k}_cs_ms"] = float(np.median(sum(times[k], [])))
                res[f"{key}_{k}_cs_spread_ms"] = max(med) - min(med)
            ev = [_lib.TrackerEvent.from_buffer_copy(bytes(row)) for row in arms["view"][2].cpu().numpy().reshape(N, rec_bytes)]
            res[f"{key}_cs_streams"] = sum(e.detection == 2 for e in ev)

            from torch.profiler import ProfilerActivity, profile
            for k, kernel in (("view", "k_feed_draw_view"), ("plain", "k_feed_draw_yuv" if fmt == "nv12" else "k_feed_draw")):
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(steps):
                        now[0] += 20.0
                        arms[k][1]()
                    torch.cuda.synchronize()
                us = 0.0
                for e in prof.key_averages():
                    if e.key.split("(")[0].split("<")[0].endswith(kernel):
                        t = getattr(e, "device_time_total", None)
                        us += t if t is not None else e.cuda_time_total
                ms = us / 1000.0 / steps
                res[f"{kernel}_{key}_ms"] = ms
            # bytes a view draw needs at least: the video it samples read once (the crop of each plane) + the canvas
            ms = res[f"k_feed_draw_view_{key}_ms"]
            video_bytes = N * sw * sh * (4 if fmt == "rgba" else 1.5)
            res[f"k_feed_draw_view_{key}_tb_per_s"] = (video_bytes + N * CW * CH * 4) / (ms * 1e-3) / 1e12 if ms > 0 else None
            for c, _, _ in arms.values():
                c.close()
            del vid, plain, keep, staged
            torch.cuda.empty_cache()
        del up
        torch.cuda.empty_cache()
    res["views_records_agree"] = True
    return res


def migrate_arms(torch, frames, stream, N, W, H, steps, rounds):
    """Tracker records (ht_tracker_export / ht_tracker_import) of N streams in steady tracking, W x H video on W/2 x H/2
    canvases, CUDA events on the library's stream around each call, repeated `rounds` x `steps` times:

      migrate_d2d       export of every stream into device memory + import of those records into a second context
      migrate_host      the same through pinned host memory (export returns after the records have landed; import
                        stages them on the device, checks them, synchronises and scatters)
      tick_before / tick_after   one steady-state ht_tracker_feed tick of the source context and of the destination
                        after the import, alternating arm by arm: a migrated stream keeps its track() scheduling history
                        (the d_track_cost words travel), so its tier placement should cost nothing

    Achieved bytes/s: N * HT_TRACKER_RECORD_BYTES per direction (written by export, read by import's check and again
    by its scatter; the model-histogram reads and writes on the device side are the same size again).  The records of
    the two contexts' ticks must agree."""
    import ctypes as C
    from headtrackr_b200 import Context, _lib
    R = _lib.TRACKER_RECORD_BYTES
    CW, CH = W // 2, H // 2
    rec_bytes = C.sizeof(_lib.TrackerEvent)
    now = [1.0e12]
    arr = (_lib.VideoFrame * N)()
    for k in range(N):
        arr[k] = _lib.VideoFrame(frames[k].data_ptr(), k, W, H, 0, 0.0)
    src = Context(max_width=CW, max_height=CH, max_frames=N, stream=stream)
    dst = Context(max_width=CW, max_height=CH, max_frames=N, stream=stream)
    for c in (src, dst):
        c.tracker_config(calcAngles=True)
    src.tracker_start(0, N)
    outs = {c: torch.empty(N * rec_bytes, dtype=torch.uint8, device="cuda") for c in (src, dst)}

    def tick(c):
        for k in range(N):
            arr[k].now_ms = now[0]
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        c._check(c._L.ht_tracker_feed(c._h, C.addressof(arr), N, 1, CW, CH, outs[c].data_ptr()))
        b.record()
        b.synchronize()
        return a.elapsed_time(b)

    for _ in range(20):                          # the whitebalance gate, detection, the first CS frames
        now[0] += 20.0
        tick(src)
    ids = (C.c_int32 * N)(*range(N))
    dev = torch.empty((N, R), dtype=torch.uint8, device="cuda")
    host = torch.empty((N, R), dtype=torch.uint8, pin_memory=True)

    def timed_call(fn):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        return a.elapsed_time(b)

    def exp(ptr):
        return lambda: src._check(src._L.ht_tracker_export(src._h, C.addressof(ids), N, ptr))

    def imp(ptr):
        return lambda: dst._check(dst._L.ht_tracker_import(dst._h, C.addressof(ids), N, ptr))

    t = {k: [] for k in ("export_d2d", "import_d2d", "export_host", "import_host", "tick_before", "tick_after")}
    for _ in range(3):                           # warm-up of both paths
        exp(dev.data_ptr())(), imp(dev.data_ptr())(), exp(host.data_ptr())(), imp(host.data_ptr())()
    for _ in range(rounds * steps):
        t["export_d2d"].append(timed_call(exp(dev.data_ptr())))
        t["import_d2d"].append(timed_call(imp(dev.data_ptr())))
        t["export_host"].append(timed_call(exp(host.data_ptr())))
        t["import_host"].append(timed_call(imp(host.data_ptr())))
    mismatches = 0
    for _ in range(rounds * steps):              # both contexts hold the same streams: tick them alternately
        now[0] += 20.0
        t["tick_before"].append(tick(src))
        t["tick_after"].append(tick(dst))
        mismatches += int(not torch.equal(outs[src], outs[dst]))
    if mismatches:
        raise SystemExit(f"migrated streams disagree with the source on {mismatches} ticks")
    res = {f"{k}_ms": float(np.median(v)) for k, v in t.items()}
    res.update({f"{k}_min_ms": float(min(v)) for k, v in t.items()})
    nbytes = N * R
    res["record_bytes"], res["migrate_bytes"] = R, nbytes
    for k in ("export_d2d", "import_d2d", "export_host", "import_host"):
        res[f"{k}_GBps"] = nbytes / (res[f"{k}_ms"] * 1e-3) / 1e9
    ev = [_lib.TrackerEvent.from_buffer_copy(bytes(row)) for row in outs[dst].cpu().numpy().reshape(N, rec_bytes)]
    res["migrate_cs_streams"] = sum(e.detection == 2 for e in ev)
    res["migrate_records_agree"] = True
    src.close()
    dst.close()
    return res


def framing_arms(torch, stream, N, steps, rounds, before_lib=None):
    """f15's workload (N streams of 1280x720 NV12 through ht_tracker_feed_yuv onto 320x240 canvases, 224x224 NV12 face
    crops on every stream), with arms alternating tick by tick: framing off (framingoff_cs), framing off on another
    build (framingoff_before_cs, --before-lib), a framing on every stream (framingall_cs) and on every 64th stream
    (framing64_cs), alpha 0.25 and dead zone 0.1.  The records of every arm must agree on every timed tick, and the
    framed arms' boxes must equal headtrackr_b200.framing's replay of the records on a sample of streams."""
    import ctypes as C
    from headtrackr_b200 import Context, _lib, framing
    from headtrackr_b200.context import _yuv_image
    W, H, CW, CH, S = 1280, 720, 320, 240, 224
    rec_bytes = C.sizeof(_lib.TrackerEvent)
    now = [1.0e12]
    kw = dict(max_width=CW, max_height=CH, max_frames=N, stream=stream)
    ys, uvs = nv12_streams(torch, N, W, H)
    keep = []
    imgs = [_yuv_image((ys[k], uvs[k]), "nv12", "bt601", keep)[0] for k in range(N)]
    yrecs = (_lib.YuvFrame * N)()
    for k in range(N):
        yrecs[k] = _lib.YuvFrame(imgs[k], k, CW, CH, 0, 0.0)
    boxes = {}

    def arm(every, before=False):
        c = other_build_context(before_lib, **kw) if before else Context(**kw)
        c._L.ht_tracker_set_face_crop_yuv.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        c.tracker_config()
        c.tracker_reset(0, N)
        c.tracker_start(0, N)
        y = torch.zeros((N, S, S), dtype=torch.uint8, device="cuda")
        uv = torch.zeros((N, S // 2, S), dtype=torch.uint8, device="cuda")
        c.tracker_set_face_crop(0, [{"out": (y[k], uv[k]), "format": "nv12", "color": "bt601"} for k in range(N)])
        if every:
            b = torch.zeros((N, 64), dtype=torch.uint8, device="cuda")
            c.tracker_set_framing(0, [{"out": b[k, :48]} if k % every == 0 else None for k in range(N)])
            boxes[every] = b
        out = torch.empty(N * rec_bytes, dtype=torch.uint8, device="cuda")

        def run():
            for k in range(N):
                yrecs[k].now_ms = now[0]
            c._check(c._L.ht_tracker_feed_yuv(c._h, C.addressof(yrecs), N, 1, out.data_ptr()))
        return c, run, out

    arms = {"framingoff_cs": arm(0), "framingall_cs": arm(1), "framing64_cs": arm(64)}
    if before_lib:
        arms["framingoff_before_cs"] = arm(0, before=True)
    names = list(arms)
    sample = list(range(0, N, max(1, N // 32)))
    replay = {k: framing.new_box() for k in sample}

    def tick(name):
        _, run, _ = arms[name]
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        run()
        b.record()
        b.synchronize()
        return a.elapsed_time(b)

    def follow():
        recs = arms["framingoff_cs"][2].cpu().numpy().reshape(N, rec_bytes)
        for k in sample:
            e = _lib.TrackerEvent.from_buffer_copy(bytes(recs[k]))
            framing.framing_step(replay[k], dict(detection=e.detection, x=e.x, y=e.y, width=e.width, height=e.height,
                                                 angle=e.angle), CW, CH)

    for _ in range(17):                          # the whitebalance gate, detection, the first CS frames
        now[0] += 20.0
        for name in names:
            tick(name)
        follow()
    times = {name: [[] for _ in range(rounds)] for name in names}
    for r in range(rounds):
        for s in range(steps):
            now[0] += 20.0
            rot = (r * steps + s) % len(names)
            for name in names[rot:] + names[:rot]:
                times[name][r].append(tick(name))
            first = arms[names[0]][2]
            if any(not torch.equal(first, arms[name][2]) for name in names[1:]):
                raise SystemExit("framing arms disagree on the records of a timed tick")
            follow()
    res = {}
    for name in names:
        med = [float(np.median(t)) for t in times[name]]
        res[f"{name}_ms"] = float(np.median(sum(times[name], [])))
        res[f"{name}_spread_ms"] = max(med) - min(med)
    res["framing_records_agree"] = True
    got = boxes[1].cpu().numpy()
    res["framing_boxes_equal_replay"] = all(bytes(got[k, :48]) == framing.box_to_bytes(replay[k]) for k in sample)
    res["framing_updates_max"] = max(replay[k]["updates"] for k in sample)
    for c, _, _ in arms.values():
        c.close()
    return res


def redact_arms(torch, stream, N, steps, rounds, before_lib=None):
    """N streams of 1280x720 NV12 through ht_tracker_feed_yuv onto 320x240 canvases, with arms alternating tick by
    tick: redaction off (redactoff_cs), off on another build (redactoff_before_cs, --before-lib), a mosaic (B = 16,
    scale 1.5) on every stream (redactall_cs) and on every 64th stream (redact64_cs).  The redaction writes the video,
    so every arm has its own copy, restored from the pristine planes before each tick, outside the timed window.  The
    records of every arm must agree on every timed tick."""
    import ctypes as C
    from headtrackr_b200 import Context, _lib
    from headtrackr_b200.context import _yuv_image
    W, H, CW, CH = 1280, 720, 320, 240
    rec_bytes = C.sizeof(_lib.TrackerEvent)
    now = [1.0e12]
    kw = dict(max_width=CW, max_height=CH, max_frames=N, stream=stream)
    ys, uvs = nv12_streams(torch, N, W, H)

    def arm(every, before=False):
        c = other_build_context(before_lib, **kw) if before else Context(**kw)
        c.tracker_config()
        c.tracker_reset(0, N)
        c.tracker_start(0, N)
        if every:
            c.tracker_set_redact(0, [{"mode": "mosaic", "block": 16, "scale": 1.5} if k % every == 0 else None
                                     for k in range(N)])
        y, uv = [t.clone() for t in ys], [t.clone() for t in uvs]
        keep = []
        imgs = [_yuv_image((y[k], uv[k]), "nv12", "bt601", keep)[0] for k in range(N)]
        recs = (_lib.YuvFrame * N)()
        for k in range(N):
            recs[k] = _lib.YuvFrame(imgs[k], k, CW, CH, 0, 0.0)
        out = torch.empty(N * rec_bytes, dtype=torch.uint8, device="cuda")

        def restore():
            for k in range(N):
                y[k].copy_(ys[k])
                uv[k].copy_(uvs[k])

        def run():
            for k in range(N):
                recs[k].now_ms = now[0]
            c._check(c._L.ht_tracker_feed_yuv(c._h, C.addressof(recs), N, 1, out.data_ptr()))
        return c, run, out, restore, (y, uv, keep)

    arms = {"redactoff_cs": arm(0), "redactall_cs": arm(1), "redact64_cs": arm(64)}
    if before_lib:
        arms["redactoff_before_cs"] = arm(0, before=True)
    names = list(arms)

    def tick(name):
        _, run, _, restore, _ = arms[name]
        restore()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        run()
        b.record()
        b.synchronize()
        return a.elapsed_time(b)

    for _ in range(17):                          # the whitebalance gate, detection, the first CS frames
        now[0] += 20.0
        for name in names:
            tick(name)
    times = {name: [[] for _ in range(rounds)] for name in names}
    for r in range(rounds):
        for s in range(steps):
            now[0] += 20.0
            rot = (r * steps + s) % len(names)
            for name in names[rot:] + names[:rot]:
                times[name][r].append(tick(name))
            first = arms[names[0]][2]
            if any(not torch.equal(first, arms[name][2]) for name in names[1:]):
                raise SystemExit("redaction arms disagree on the records of a timed tick")
    res = {}
    for name in names:
        med = [float(np.median(t)) for t in times[name]]
        res[f"{name}_ms"] = float(np.median(sum(times[name], [])))
        res[f"{name}_spread_ms"] = max(med) - min(med)
    res["redact_records_agree"] = True
    y = arms["redactall_cs"][4][0]
    res["redact_streams_changed"] = sum(int(not torch.equal(y[k], ys[k])) for k in range(N))
    for c, _, _, _, _ in arms.values():
        c.close()
    return res


def best_shot_arms(torch, stream, N, steps, rounds, before_lib=None):
    """f15's workload (N streams of 1280x720 NV12 through ht_tracker_feed_yuv onto 320x240 canvases, 224x224 NV12 face
    crops on every stream), with arms alternating tick by tick: no best shot (bestoff_cs), none on another build
    (bestoff_before_cs, --before-lib), a 224x224 best shot with two images on every stream (bestall_cs) and on every
    64th stream (best64_cs).  The records of every arm must agree on every timed tick, and the states of a sample of
    streams must equal headtrackr_b200.bestshot's replay of the records and the host score of the images' candidates.
    Then, in runs of their own under torch.profiler, the kernel times of k_best_score and k_best_write per tick."""
    import ctypes as C
    from headtrackr_b200 import Context, _lib, bestshot
    from headtrackr_b200.context import _yuv_image
    W, H, CW, CH, S = 1280, 720, 320, 240, 224
    rec_bytes = C.sizeof(_lib.TrackerEvent)
    now = [1.0e12]
    kw = dict(max_width=CW, max_height=CH, max_frames=N, stream=stream)
    ys, uvs = nv12_streams(torch, N, W, H)
    keep = []
    imgs = [_yuv_image((ys[k], uvs[k]), "nv12", "bt601", keep)[0] for k in range(N)]
    yrecs = (_lib.YuvFrame * N)()
    for k in range(N):
        yrecs[k] = _lib.YuvFrame(imgs[k], k, CW, CH, 0, 0.0)
    shots = {}

    def arm(every, before=False):
        c = other_build_context(before_lib, **kw) if before else Context(**kw)
        c._L.ht_tracker_set_face_crop_yuv.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        c.tracker_config()
        c.tracker_reset(0, N)
        c.tracker_start(0, N)
        y = torch.zeros((N, S, S), dtype=torch.uint8, device="cuda")
        uv = torch.zeros((N, S // 2, S), dtype=torch.uint8, device="cuda")
        c.tracker_set_face_crop(0, [{"out": (y[k], uv[k]), "format": "nv12", "color": "bt601"} for k in range(N)])
        if every:
            img = torch.zeros((N, 2, S, S, 4), dtype=torch.uint8, device="cuda")
            st = torch.zeros((N, 128), dtype=torch.uint8, device="cuda")
            c.tracker_set_best_shot(0, [{"out": (img[k, 0], img[k, 1]), "state": st[k, :96]} if k % every == 0 else None
                                        for k in range(N)])
            shots[every] = (img, st)
        out = torch.empty(N * rec_bytes, dtype=torch.uint8, device="cuda")

        def run():
            for k in range(N):
                yrecs[k].now_ms = now[0]
            c._check(c._L.ht_tracker_feed_yuv(c._h, C.addressof(yrecs), N, 1, out.data_ptr()))
        return c, run, out

    arms = {"bestoff_cs": arm(0), "bestall_cs": arm(1), "best64_cs": arm(64)}
    if before_lib:
        arms["bestoff_before_cs"] = arm(0, before=True)
    names = list(arms)
    sample = list(range(0, N, max(1, N // 32)))
    replay = {k: bestshot.new_state() for k in sample}
    candidate = {}

    def tick(name):
        _, run, _ = arms[name]
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        run()
        b.record()
        b.synchronize()
        return a.elapsed_time(b)

    def follow():
        # a written image is the candidate of a best tick: its score is the state's best_score when it was written
        recs = arms["bestoff_cs"][2].cpu().numpy().reshape(N, rec_bytes)
        img, st = shots[1]
        states = st.cpu().numpy()
        for k in sample:
            e = _lib.TrackerEvent.from_buffer_copy(bytes(recs[k]))
            r = dict(detection=e.detection, x=e.x, y=e.y, width=e.width, height=e.height, angle=e.angle)
            got = bestshot.state_from_bytes(states[k, :96])
            score = got["score"] if bestshot.crop_tick(r) else 0
            if bestshot.step(replay[k], r, score, now[0], CW, CH):
                candidate[k] = bestshot.score(img[k, replay[k]["buffer"]].cpu().numpy())
            if bestshot.state_to_bytes(replay[k]) != bytes(states[k, :96]) or \
                    (k in candidate and candidate[k] != replay[k]["best_score"]):
                raise SystemExit(f"best-shot state or image of stream {k} disagrees with the replay")

    for _ in range(17):                          # the whitebalance gate, detection, the first CS frames
        now[0] += 20.0
        for name in names:
            tick(name)
        follow()
    times = {name: [[] for _ in range(rounds)] for name in names}
    for r in range(rounds):
        for s in range(steps):
            now[0] += 20.0
            rot = (r * steps + s) % len(names)
            for name in names[rot:] + names[:rot]:
                times[name][r].append(tick(name))
            first = arms[names[0]][2]
            if any(not torch.equal(first, arms[name][2]) for name in names[1:]):
                raise SystemExit("best-shot arms disagree on the records of a timed tick")
            follow()
    res = {}
    for name in names:
        med = [float(np.median(t)) for t in times[name]]
        res[f"{name}_ms"] = float(np.median(sum(times[name], [])))
        res[f"{name}_spread_ms"] = max(med) - min(med)
    res["best_records_agree"] = True
    res["best_states_equal_replay"] = True
    res["best_tracks_max"] = max(replay[k]["track"] for k in sample)
    res["best_improved_ticks_sampled"] = sum(replay[k]["best_tick"] for k in sample)

    from torch.profiler import ProfilerActivity, profile
    for name in ("bestall_cs", "best64_cs"):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(steps):
                now[0] += 20.0
                arms[name][1]()
            torch.cuda.synchronize()
        for kern in ("k_best_score", "k_best_write", "k_face_crop"):
            us = 0.0
            for e in prof.key_averages():
                if kern in e.key:
                    t = getattr(e, "device_time_total", None)
                    us += t if t is not None else e.cuda_time_total
            res[f"{kern}_{name[:-3]}_ms"] = us / 1000.0 / steps
    for c, _, _ in arms.values():
        c.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5, help="rounds of the alternating feed arms (their spread)")
    ap.add_argument("--before-lib", help="another build of libheadtrackr_b200.so for the one-size feed arm")
    ap.add_argument("--only-canvases", action="store_true", help="only the canvas arms (canvas_arms)")
    ap.add_argument("--debug-streams", action="store_true", help="only the debug-canvas arms (debug_arms)")
    ap.add_argument("--strokes", action="store_true", help="only the debug-stroke arms (strokes_arms)")
    ap.add_argument("--migrate", action="store_true", help="only the tracker-record arms (migrate_arms)")
    ap.add_argument("--camera-streams", action="store_true", help="only the camera-controller arms (camera_arms)")
    ap.add_argument("--yuv", action="store_true", help="only the YUV video arms (yuv_arms)")
    ap.add_argument("--formats", action="store_true", help="only the video-format arms (formats_arms)")
    ap.add_argument("--views", action="store_true", help="only the video-view arms (views_arms)")
    ap.add_argument("--crops", action="store_true", help="only the face-crop arms (crops_arms)")
    ap.add_argument("--framing", action="store_true", help="only the framing arms (framing_arms)")
    ap.add_argument("--redact", action="store_true", help="only the face-redaction arms (redact_arms)")
    ap.add_argument("--best-shot", action="store_true", help="only the best-shot arms (best_shot_arms)")
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch
    from headtrackr_b200 import Context, synth
    N, W, H = a.streams, 640, 480
    base = np.stack([synth.frame(i, W, H, n_faces=1) for i in range(8)])
    frames = torch.from_numpy(np.ascontiguousarray(base[np.arange(N) % 8])).cuda()
    res = dict(streams=N, width=W, height=H, steps=a.steps)
    res["gpu"], res["power_limit"] = gpu_info()

    ts = torch.cuda.Stream()                # the library runs on this stream and the events below are recorded on it
    torch.cuda.set_stream(ts)
    stream = ts.cuda_stream
    if a.yuv:
        res.update(yuv_arms(torch, stream, N, a.steps, a.rounds, a.before_lib))
        return report(res, a.out)
    if a.views:
        res.update(views_arms(torch, stream, N, a.steps, a.rounds, a.before_lib))
        return report(res, a.out)
    if a.crops:
        res.update(crops_arms(torch, stream, N, a.steps, a.rounds, a.before_lib))
        return report(res, a.out)
    if a.framing:
        res.update(framing_arms(torch, stream, N, a.steps, a.rounds, a.before_lib))
        return report(res, a.out)
    if a.redact:
        res.update(redact_arms(torch, stream, N, a.steps, a.rounds, a.before_lib))
        return report(res, a.out)
    if a.best_shot:
        res.update(best_shot_arms(torch, stream, N, a.steps, a.rounds, a.before_lib))
        return report(res, a.out)
    if a.formats:
        res.update(formats_arms(torch, stream, N, a.steps, a.rounds, a.before_lib))
        return report(res, a.out)
    if a.migrate:
        res.update(migrate_arms(torch, frames, stream, N, W, H, a.steps, a.rounds))
        return report(res, a.out)
    if a.camera_streams:
        res.update(camera_arms(torch, frames, stream, N, W, H, a.steps, a.rounds, a.before_lib))
        return report(res, a.out)
    if a.strokes:
        res.update(strokes_arms(torch, frames, stream, N, W, H, a.steps, a.rounds, a.before_lib))
        return report(res, a.out)
    if a.debug_streams:
        res.update(debug_arms(torch, frames, stream, N, W, H, a.steps, a.rounds, a.before_lib))
        return report(res, a.out)
    if a.only_canvases:
        res.update(canvas_arms(torch, frames, stream, N, W, H, a.steps, a.rounds, a.before_lib))
        return report(res, a.out)
    c = Context(max_width=W, max_height=H, max_frames=N, stream=stream)
    ev = torch.empty(N * 144, dtype=torch.uint8, device="cuda")
    c.tracker_config()
    c.tracker_reset(0, N)
    c.tracker_start(0, N)
    now = [1.0e12]

    def tick():
        now[0] += 20.0
        c.tracker_step(frames, now[0], out=ev)
    c.sync()
    res["tracker_wb_ms"] = timed(torch, tick, min(a.steps, 13))[0]      # frames 1..13 of the 15-sample gate
    for _ in range(4):                                                  # rest of the gate, detection, first CS frames
        tick()
    c.sync()
    res["tracker_cs_ms"] = timed(torch, tick, a.steps)[0]
    res["tracker_cs_streams"] = sum(r["detection"] == "CS" for r in c.tracker_step(frames, now[0] + 20.0))
    c.tracker_config(enable=False)
    c.close()

    c = Context(max_width=W, max_height=H, max_frames=N, stream=stream)
    c.stream_head_config()
    c.stream_reset(0, N)
    import ctypes as C
    from headtrackr_b200 import _lib
    sev = torch.empty(N * C.sizeof(_lib.StreamEvent), dtype=torch.uint8, device="cuda")
    hev = torch.empty(N * C.sizeof(_lib.HeadEvent), dtype=torch.uint8, device="cuda")

    def step_head():
        c._check(c._L.ht_stream_step_head(c._h, frames.data_ptr(), N, W, H, 5, 1, 0, sev.data_ptr(), hev.data_ptr()))
    for _ in range(3):
        step_head()
    c.sync()
    res["stream_head_cs_ms"] = timed(torch, step_head, a.steps)[0]
    res["stream_head_cs_streams"] = sum(e["detection"] == "CS" for e in c.stream_step_head(frames)[0])
    c.close()
    res.update(feed_arms(torch, frames, stream, N, W, H, a.steps, a.rounds))
    res.update(canvas_arms(torch, frames, stream, N, W, H, a.steps, a.rounds, a.before_lib))
    report(res, a.out)


def report(res, out):
    line = json.dumps(res)
    print(line)
    if out:
        Path(out).parent.mkdir(parents=True, exist_ok=True)
        Path(out).write_text(line + "\n")


if __name__ == "__main__":
    main()
