#!/usr/bin/env python
"""CPU model of k_track's launch schedule (strict mode: every mean-shift pass summed).

Per-stream work comes from the CPU oracle (passes per call and window sizes of the bench mix); the time of a pass on a
cluster of c CTAs is read off single-stream chain times (PX_T / US below, from tools/track_chain_probe.py); the GPU
is 3 * SMS CTA slots (3 CTAs of 256 threads per SM) filled strictly in launch order, as the block scheduler does.  Prints the makespan of a few launch orders / cluster assignments to rank ideas for the
streams whose chains end last.

    python tools/track_schedule_model.py [n_streams]
"""
import math
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import oracle  # noqa: E402  (analysis tool, not the product)
from headtrackr_b200 import synth  # noqa: E402

SMS = 132              # H100 SXM
W, H, CALLS, SLOTS = 640, 480, 30, 3 * SMS
# microseconds per pass vs pixels per thread, one stream alone (frame 58 at 1/2/4/8 CTAs; a whole-frame window at 2).
# Taken on an earlier GPU and not re-measured on H100: re-run tools/track_chain_probe.py there before trusting
# absolute makespans (the model ranks launch orders, which depend mostly on the shape of this curve).
PX_T = [0, 24, 48, 96, 192, 600, 1200]
US = [2.6, 3.4, 4.65, 6.6, 8.85, 16.0, 30.0]
LOAD_FACTOR = 1.3      # passes are ~30 % slower when every SM holds 3 busy CTAs (timeline vs probe)


def stream_work(j, blob):
    base = synth.frame(j % 64, W, H)
    f = np.roll(base, (j // 64) * 16, axis=1)
    res = oracle.detect(f, blob)
    if not res:
        return None
    best = res[0]
    for r in res[1:]:
        if r[4] > best[4]:
            best = r
    if not best[4] > -10:
        return None
    ot = oracle.CamshiftTracker(calc_angles=False)
    ot.init_tracker(f, *[int(math.floor(v)) for v in best[:4]])
    passes = []
    for _ in range(CALLS):
        sx, sy, sw, sh = ot.search_window()
        tr = ot.track(f)
        x0, y0 = max(sx, 0), max(sy, 0)
        px = max(0, min(x0 + sw, W) - x0) * max(0, min(y0 + sh, H) - y0)
        passes.append((int(tr.n_iter), px))
    first = passes[0][1]
    return first, passes


def stream_time(passes, c):
    t = 0.0
    for n_iter, px in passes:
        t += n_iter * float(np.interp(px / (256.0 * c), PX_T, US))
    return t * LOAD_FACTOR


def makespan(order, clusters, times):
    """strictly in-order placement of clusters on SLOTS CTA slots"""
    import heapq
    free_at = [0.0] * SLOTS      # min-heap of slot release times
    heapq.heapify(free_at)
    end = 0.0
    for i in order:
        c = clusters[i]
        ts = [heapq.heappop(free_at) for _ in range(c)]
        start = max(ts)
        fin = start + times[i][c]
        for _ in range(c):
            heapq.heappush(free_at, fin)
        end = max(end, fin)
    return end


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 1024
    blob = synth.load_cascade_blob()
    oracle.lib()
    with ThreadPoolExecutor(max_workers=8) as ex:
        work = list(ex.map(lambda j: stream_work(j, blob), range(n)))
    idx = [i for i, w in enumerate(work) if w is not None]
    print(f"{len(idx)} of {n} streams found a face")
    times = {i: {c: stream_time(work[i][1], c) for c in (1, 2, 4, 8)} for i in idx}
    area0 = {i: work[i][0] for i in idx}
    npass = np.array([sum(p[0] for p in work[i][1]) for i in idx])
    print(f"passes per stream: mean {npass.mean():.1f} p50 {np.median(npass):.0f} p90 {np.percentile(npass, 90):.0f} max {npass.max()}")
    t2 = np.array([times[i][2] for i in idx])
    print(f"chain at 2 CTAs (us): mean {t2.mean():.0f} p90 {np.percentile(t2, 90):.0f} max {t2.max():.0f};  sum/222 slots = {t2.sum() / 222:.0f} us")
    by_index = idx
    by_area = sorted(idx, key=lambda i: -area0[i])
    by_cost = sorted(idx, key=lambda i: -times[i][2])

    def all_c(c):
        return {i: c for i in idx}
    rows = [("index order, 2 CTAs", by_index, all_c(2)),
            ("largest initial window first, 2 CTAs   (round-1 default)", by_area, all_c(2)),
            ("true cost first, 2 CTAs                 (cost known: lower bound for ordering alone)", by_cost, all_c(2)),
            ("true cost first, 4 CTAs", by_cost, all_c(4)),
            ("true cost first, 1 CTA", by_cost, all_c(1))]
    for k in (8, 16, 32, 64, 128):
        cl = all_c(2)
        for i in by_cost[:k]:
            cl[i] = 8
        rows.append((f"true cost first, the {k} costliest streams on 8 CTAs, rest 2", by_cost, cl))
    for k in (32, 128):
        cl = all_c(2)
        for i in by_cost[:k]:
            cl[i] = 4
        rows.append((f"true cost first, the {k} costliest streams on 4 CTAs, rest 2", by_cost, cl))
    cl = all_c(1)
    for i in by_cost[:128]:
        cl[i] = 8
    rows.append(("true cost first, 128 costliest on 8 CTAs, rest 1 CTA", by_cost, cl))
    for name, order, cl in rows:
        print(f"{makespan(order, cl, times) / 1e3:7.2f} ms   {name}")
    # history-free two-phase launch: phase A = the first K calls of every stream (2 CTAs, area order) also measures each
    # stream's cost; phase B = the remaining calls, costliest-so-far first, the top streams on 8 CTAs
    for K in (2, 3, 5):
        ta = {i: {c: stream_time(work[i][1][:K], c) for c in (1, 2, 4, 8)} for i in idx}
        tb = {i: {c: stream_time(work[i][1][K:], c) for c in (1, 2, 4, 8)} for i in idx}
        a_ms = makespan(by_area, all_c(2), ta)
        pred = sorted(idx, key=lambda i: -ta[i][2])
        for k in (16, 32, 64):
            cl = all_c(2)
            for i in pred[:k]:
                cl[i] = 8
            b_ms = makespan(pred, cl, tb)
            print(f"{(a_ms + b_ms) / 1e3:7.2f} ms   two-phase: {K} calls to measure ({a_ms / 1e3:.2f}), then by measured cost, top {k} on 8 CTAs ({b_ms / 1e3:.2f})")


if __name__ == "__main__":
    main()
