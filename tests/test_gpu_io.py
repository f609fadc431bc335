"""GPU: caller buffers and context lifetime.

  * I/O matrix: every entry point that takes caller buffers gives byte-identical results, and the same number of kernel
    launches, whichever of its buffers are host memory (numpy) and which device memory (torch CUDA), with each optional
    output present or NULL.  Every combination runs the same seeded inputs on a fresh context.
  * Lifecycle: a context that has made every resource it creates on first use (copy, aux, pyramid and tier streams,
    their events, the pinned feed table, the head state, profiling events) closes cleanly; twice in one process, with
    identical results and no device memory left behind by the first round."""
import ctypes as C
import itertools

import numpy as np
import pytest

from headtrackr_b200 import Context, synth
from headtrackr_b200._lib import VideoFrame

pytestmark = pytest.mark.gpu

W, H, N = 320, 240, 4
FR = synth.batch(N, W, H)
RECT, TOBJ, WIN, SEV, HEV, TEV = 48, 24, 16, 56, 64, 144
SLOTS = np.array([5, 1, 0, 2], np.int32)      # a permutation, so that slot != frame
WHERE = ("host", "dev")


def put(a, where):
    """a caller buffer holding the bytes of `a`: the numpy array itself (host) or a torch CUDA copy (dev)"""
    a = np.ascontiguousarray(a)
    if where == "host":
        return a
    import torch
    return torch.from_numpy(a.copy()).cuda()


def out(where, nbytes):
    return None if where is None else put(np.zeros(nbytes, np.uint8), where)


def ptr(b):
    return None if b is None else (b.ctypes.data if isinstance(b, np.ndarray) else b.data_ptr())


def read(b):
    return None if b is None else (b if isinstance(b, np.ndarray) else b.cpu().numpy()).tobytes()


def unpad(data, size, pad):
    """records of `size` bytes with the padding bytes [pad[0], pad[1]) zeroed (the kernels do not write them)"""
    a = np.frombuffer(data, np.uint8).reshape(-1, size).copy()
    a[:, pad[0]:pad[1]] = 0
    return a.tobytes()


def detections(rects, counts, n=N, K=64):
    """the rect lists: only the first counts[f] records of each frame are results"""
    c = np.frombuffer(counts, np.int32)
    r = np.frombuffer(unpad(rects, RECT, (44, 48)), np.uint8).reshape(n, K * RECT)
    return c.tobytes() + b"".join(r[f, :RECT * min(int(c[f]), K)].tobytes() for f in range(n))


def call(ctx, fn, *outs):
    """-> (kernel launches of the call, the outputs' bytes after the call has finished)"""
    import torch
    torch.cuda.synchronize()                   # device inputs are in place (the library runs on its own stream)
    before = ctx.launch_count
    ctx._check(fn())
    launches = ctx.launch_count - before
    ctx.sync()
    return launches, [read(o) for o in outs]


def fresh(max_frames=8):
    return Context(max_width=W, max_height=H, max_frames=max_frames)


def model(ctx, slots):
    return [ctx.debug_model_hist(int(s)).tobytes() for s in slots]


def host_track(ctx, slots=None):
    objs, wins = ctx.track(FR, slots=None if slots is None else [int(s) for s in slots], n_calls=2)
    return repr((objs, wins))


# ---- one runner per entry point: variant -> (launches, [results]); None marks an absent optional output ----

def run_detect(v):
    fr, o_r, o_c = v
    ctx = fresh()
    L = ctx._L
    frames, rects, counts = put(FR, fr), out(o_r, N * ctx.K * RECT), out(o_c, 4 * N)
    n, res = call(ctx, lambda: L.ht_detect(ctx._h, ptr(frames), N, W, H, 5, 1, ptr(rects), ptr(counts)), rects, counts)
    ctx.close()
    return n, [detections(res[0], res[1], K=ctx.K)]


def seed_rects():
    return np.array([[110, 60, 90, 110]] * N, np.int32)


def run_track_init(v):
    fr, rc, sl = v
    ctx = fresh()
    L = ctx._L
    frames, rects, slots = put(FR, fr), put(seed_rects(), rc), None if sl is None else put(SLOTS, sl)
    used = SLOTS if sl is not None else np.arange(N)
    n, _ = call(ctx, lambda: L.ht_track_init(ctx._h, ptr(slots), N, ptr(frames), W, H, ptr(rects), 1))
    res = [b"".join(model(ctx, used)), host_track(ctx, used)]
    ctx.close()
    return n, res


def run_track_init_from_detect(v):
    fr, dr, dc, fo = v
    ctx = fresh()
    L = ctx._L
    rects, counts = ctx.detect_raw(FR)
    det_r = put(np.frombuffer(bytes(rects), np.uint8), dr)
    det_c = put(np.frombuffer(bytes(counts), np.uint8), dc)
    frames, found = put(FR, fr), out(fo, 4 * N)
    n, res = call(ctx, lambda: L.ht_track_init_from_detect(ctx._h, None, N, ptr(frames), W, H, ptr(det_r), ptr(det_c), 0,
                                                           ptr(found)), found)
    res += [b"".join(model(ctx, range(N))), host_track(ctx)]
    ctx.close()
    return n, res


def run_track(v):
    fr, ob, wi = v
    ctx = fresh()
    L = ctx._L
    ctx.track_init(FR, seed_rects())
    frames, objs, wins = put(FR, fr), out(ob, N * TOBJ), out(wi, N * WIN)
    n, res = call(ctx, lambda: L.ht_track(ctx._h, None, N, ptr(frames), W, H, 3, ptr(objs), ptr(wins)), objs, wins)
    ctx.close()
    return n, res


def run_detect_track(v):
    fr, o_r, o_c, fo, ob, wi = v
    ctx = fresh()
    L = ctx._L
    frames = put(FR, fr)
    rects, counts, found = out(o_r, N * ctx.K * RECT), out(o_c, 4 * N), out(fo, 4 * N)
    objs, wins = out(ob, N * TOBJ), out(wi, N * WIN)
    n, res = call(ctx, lambda: L.ht_detect_track(ctx._h, ptr(frames), N, W, H, 5, 1, 0, 2, ptr(rects), ptr(counts),
                                                 ptr(found), ptr(objs), ptr(wins)), rects, counts, found, objs, wins)
    ctx.close()
    return n, [detections(res[0], res[1], K=ctx.K)] + res[2:]


def run_stream_step_head(v):
    fr, ev, hd = v
    ctx = fresh()
    L = ctx._L
    ctx.stream_head_config()
    frames = put(FR, fr)
    total, res = 0, []
    for _ in range(3):                          # VJ -> CS -> CS
        events, heads = out(ev, N * SEV), out(hd, N * HEV)
        n, r = call(ctx, lambda: L.ht_stream_step_head(ctx._h, ptr(frames), N, W, H, 5, 1, 0, ptr(events), ptr(heads)),
                    events, heads)
        total += n
        res += r
    ctx.close()
    return total, res


def tracker(ctx):
    ctx.tracker_config()
    ctx.tracker_start(0, N)


def run_tracker_step(v):
    fr, ev = v
    ctx = fresh()
    L = ctx._L
    tracker(ctx)
    frames = put(FR, fr)
    total, res = 0, []
    for t in range(4):
        events = out(ev, N * TEV)
        n, r = call(ctx, lambda: L.ht_tracker_step(ctx._h, ptr(frames), N, W, H, 1000.0 * (t + 1), ptr(events)), events)
        total += n
        res.append(unpad(r[0], TEV, (68, 72)))
    ctx.close()
    return total, res


def run_tracker_feed(v):
    fr, ev = v
    ctx = fresh()
    L = ctx._L
    tracker(ctx)
    videos = [put(synth.frame(10 + k, 400, 300), fr) for k in range(3)]
    total, res = 0, []
    for t in range(3):
        recs = (VideoFrame * 3)()
        for b, k in enumerate((2, 0, 3)):
            recs[b] = VideoFrame(ptr(videos[b]), k, 400, 300, 0, 1000.0 * (t + 1) + k)
        events = out(ev, 3 * TEV)
        n, r = call(ctx, lambda: L.ht_tracker_feed(ctx._h, C.addressof(recs), 3, int(fr == "dev"), W, H, ptr(events)),
                    events)
        total += n
        res.append(unpad(r[0], TEV, (68, 72)))
    ctx.close()
    return total, res


def run_ingest(v):
    src_where, dst_where, sw, sh = v
    ctx = fresh()
    L = ctx._L
    src = put(synth.batch(N, sw, sh, start=20), src_where)
    dst = out(dst_where, N * W * H * 4)
    n, res = call(ctx, lambda: L.ht_ingest(ctx._h, ptr(src), N, sw, sh, ptr(dst), W, H), dst)
    ctx.close()
    return n, res


def run_backprojection(v):
    fr, o = v
    ctx = fresh()
    L = ctx._L
    ctx.track_init(FR, seed_rects())
    frame, dst = put(FR[2], fr), out(o, W * H * 4)
    n, res = call(ctx, lambda: L.ht_backprojection(ctx._h, 2, ptr(frame), W, H, ptr(dst)), dst)
    ctx.close()
    return n, res


def run_whitebalance(v):
    fr, o = v
    ctx = fresh()
    L = ctx._L
    frames, dst = put(FR, fr), out(o, 8 * N)
    n, res = call(ctx, lambda: L.ht_whitebalance(ctx._h, ptr(frames), N, W, H, ptr(dst)), dst)
    ctx.close()
    return n, res


OPT = (None,) + WHERE
MATRIX = {
    "ht_detect": (run_detect, list(itertools.product(WHERE, WHERE, WHERE))),
    "ht_track_init": (run_track_init, list(itertools.product(WHERE, WHERE, OPT))),
    "ht_track_init_from_detect": (run_track_init_from_detect, list(itertools.product(WHERE, WHERE, WHERE, OPT))),
    "ht_track": (run_track, list(itertools.product(WHERE, WHERE, OPT))),
    "ht_detect_track": (run_detect_track, list(itertools.product(WHERE, WHERE, WHERE, OPT, WHERE, OPT))),
    "ht_stream_step_head": (run_stream_step_head, list(itertools.product(WHERE, WHERE, OPT))),
    "ht_tracker_step": (run_tracker_step, list(itertools.product(WHERE, WHERE))),
    "ht_tracker_feed": (run_tracker_feed, list(itertools.product(WHERE, WHERE))),
    "ht_ingest": (run_ingest, [v + g for g in ((200, 150), (W, H)) for v in itertools.product(WHERE, WHERE)]),
    "ht_backprojection": (run_backprojection, list(itertools.product(WHERE, WHERE))),
    "ht_whitebalance": (run_whitebalance, list(itertools.product(WHERE, WHERE))),
}


@pytest.mark.parametrize("entry", sorted(MATRIX))
def test_io_matrix(entry):
    run, variants = MATRIX[entry]
    results = {v: run(v) for v in variants}
    groups = {}                                  # ht_ingest: one geometry per group; otherwise one group
    for v, r in results.items():
        groups.setdefault(v[2:] if entry == "ht_ingest" else (), []).append((v, r))
    for members in groups.values():
        v0, (n0, r0) = members[0]
        for v, (n, r) in members[1:]:
            assert n == n0, (entry, v, n, v0, n0)
            assert len(r) == len(r0)
        for i in range(len(r0)):                 # output i, in every variant where it is present
            present = [(v, r[i]) for v, (n, r) in members if r[i] is not None]
            assert present, (entry, i)
            assert present[0][1], (entry, i)
            for v, data in present[1:]:
                assert data == present[0][1], (entry, i, v, present[0][0])


def lifecycle_round(monkeypatch):
    """one context touches every resource it makes on first use, then closes -> its results"""
    import torch
    monkeypatch.setenv("HT_OVERLAP", "2")        # host-frame detect_track in two parts: aux stream, part events
    monkeypatch.setenv("HT_H2D_CHUNK", "8")      # ... and several chunk events on the copy stream
    monkeypatch.setenv("HT_DETECT_PIPE", "1")    # gray + pyramid of the next wave on the pyramid stream
    monkeypatch.setenv("HT_WAVE", "4")
    n = 128                                      # ht_track of >= 128 streams runs its tiers on the tier streams
    frames = synth.batch(n, 160, 120, start=40)
    res = []
    ctx = Context(max_width=W, max_height=H, max_frames=n)
    try:
        ctx.profile(True)                        # profiling events
        dets, found, objs, wins = ctx.detect_track(frames[:64], n_calls=2)
        res.append(repr((dets, found, objs, wins)))
        ctx.set_pipeline(True)                   # pipelined detect_track: device frames and outputs
        dev = torch.from_numpy(frames[:16]).cuda()
        outs = (torch.zeros(16 * ctx.K * RECT, dtype=torch.uint8, device="cuda"),
                torch.zeros(16, dtype=torch.int32, device="cuda"), torch.zeros(16, dtype=torch.int32, device="cuda"),
                torch.zeros(16 * TOBJ, dtype=torch.uint8, device="cuda"), torch.zeros(16 * WIN, dtype=torch.uint8, device="cuda"))
        torch.cuda.synchronize()
        for _ in range(2):
            ctx.detect_track(dev, n_calls=2, outputs=outs)
        ctx.sync()
        res.append(detections(outs[0].cpu().numpy().tobytes(), outs[1].cpu().numpy().tobytes(), 16, ctx.K))
        res += [o.cpu().numpy().tobytes() for o in outs[2:]]
        ctx.set_pipeline(False)
        ctx.track_init(frames, np.array([[40, 30, 60, 60]] * n, np.int32))
        res.append(repr(ctx.track(frames, n_calls=3)))
        ctx.stream_head_config()
        res.append(repr(ctx.stream_step_head(frames[:8])))
        ctx.tracker_config()
        ctx.tracker_start(0, 8)
        res.append(repr(ctx.tracker_feed([3, 1], [frames[0], frames[1]], [1000.0, 1010.0], W, H)))
        res.append(repr(ctx.tracker_step(synth.batch(8, W, H), 2000.0)))
        prof = ctx.profile_read()
        res.append(repr({k: launches for k, (ms, launches) in prof.items()}))
        res.append(ctx.launch_count)
    finally:
        ctx.close()
    torch.cuda.synchronize()
    return res


def test_lifecycle(monkeypatch):
    import torch
    first = lifecycle_round(monkeypatch)
    torch.cuda.empty_cache()
    free_after_first = torch.cuda.mem_get_info()[0]
    second = lifecycle_round(monkeypatch)
    torch.cuda.empty_cache()
    free_after_second = torch.cuda.mem_get_info()[0]
    assert first == second
    assert free_after_second >= free_after_first - (16 << 20), (free_after_first, free_after_second)
