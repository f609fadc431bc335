"""GPU: pipelined ht_detect_track calls that change frame size, batch size or interval between calls give the results of
unpipelined ones, and of the oracle.

The tracking of pipelined call s runs on the library's second stream while call s+1's gray pass writes its bin planes
and histograms; nothing orders the two, so the slices of consecutive calls must be disjoint whatever size each call has
(DESIGN.md §5.5, tests/test_pipeline_offsets_host.py).  Each sequence runs once unpipelined (fresh outputs, a sync after
every call: the expected results) and once pipelined (one output set per call, one sync at the end), with the window
memo off and on.  Every call tracks 30 times and consecutive calls get different frames, so that call s's tracking is
long in flight under call s+1's detection and planes overwritten by the other call would change its results."""
import numpy as np
import pytest

import oracle
from headtrackr_b200 import synth
from headtrackr_b200.context import Context

pytestmark = pytest.mark.gpu

N_CALLS = 30
A, B, C_, ODD1, ODD2 = (320, 240), (160, 120), (256, 192), (161, 121), (97, 83)
X, Y = (160, 120), (128, 96)


def call(size, n, seed, interval=5, host=False, angles=True):
    """one ht_detect_track call: n frames of size from seed on; host=True: host outputs (a call that joins)"""
    return dict(w=size[0], h=size[1], n=n, seed=seed, interval=interval, host=host, angles=angles)


# name -> (context maxima (w, h, frames), calls, check the first and last call against the oracle)
SEQUENCES = {
    # A, A, B is the smallest case whose slices overlapped when a parity was cut from the call's own w * h
    "sizes": ((320, 240, 12), [call(s, 12, 100 * i) for i, s in enumerate((A, A, B, B, A, B, A, A))], True),
    "batches": ((320, 240, 12), [call(s, n, 100 * i) for i, (s, n) in
                                 enumerate(((A, 12), (C_, 7), (B, 1), (A, 12), (C_, 12), (B, 7), (A, 12)))], False),
    # odd max_frames * w * h: parity slices that are not whole multiples of 8 entries
    "odd": ((161, 121, 13), [call(s, n, 100 * i) for i, (s, n) in
                             enumerate(((ODD1, 13), (ODD2, 13), (ODD1, 5), (ODD2, 13), (ODD1, 13), (ODD2, 1)))], True),
    # a control: new plans, the same planes
    "intervals": ((320, 240, 12), [call(A, 12, 100 * i, interval=iv) for i, iv in enumerate((5, 3, 5))], False),
    # the host-output call joins and starts the parities over; the pipelined calls after it change size
    "join": ((320, 240, 12), [call(A, 12, 0), call(A, 12, 100), call(A, 12, 200, host=True), call(B, 12, 300),
                              call(B, 12, 400), call(A, 12, 500)], False),
    # >= 128 streams: k_track's three tiers on their side streams during the size change.  Without angles: the tier,
    # and so the cluster size that orders a stream's moment sums, follows the costs of the slot's earlier launches,
    # which differ between the two runs, and the fp64 angle is only pinned to the oracle's within 1e-4 (DESIGN.md §4)
    "tiers": ((160, 120, 192), [call(s, 192, 1000 * i, angles=False) for i, s in enumerate((X, X, Y, Y, X))], False),
}

_frames = {}


def frames(c):
    """(n, h, w, 4) u8: 48 distinct frames, tiled with x-rolls past 48 (the same frame at another place)"""
    key = (c["w"], c["h"], c["n"], c["seed"])
    if key not in _frames:
        f = np.stack([synth.frame(c["seed"] + i % 48, c["w"], c["h"]) for i in range(c["n"])])
        for j in range(48, c["n"]):
            f[j] = np.roll(f[j], (j // 48) * 8, axis=1)
        _frames[key] = f
    return _frames[key]


def new_outputs(torch, K, n):
    return (torch.zeros((n, K, 6), dtype=torch.float64, device="cuda"), torch.zeros((n,), dtype=torch.int32, device="cuda"),
            torch.zeros((n,), dtype=torch.int32, device="cuda"), torch.zeros((n, 6), dtype=torch.int32, device="cuda"),
            torch.zeros((n, 4), dtype=torch.int32, device="cuda"))


def host_copy(outs):
    return [o.cpu().numpy().copy() for o in outs]


def same_results(got, exp):
    """(rects, counts, found, objs, windows): rect entries beyond a frame's count are never written by the library and
    hold whatever an earlier call left there."""
    if not all(np.array_equal(a, b) for a, b in zip(got[1:], exp[1:])):
        return False
    return all(np.array_equal(got[0][f, :c], exp[0][f, :c]) for f, c in enumerate(exp[1]))


def run(torch, ctx, calls, dev, pipelined):
    """-> per call its outputs on the host: device outputs as arrays, host outputs as detect_track returns them"""
    ctx.set_pipeline(pipelined)
    res = []
    for c, d in zip(calls, dev):
        if c["host"]:
            res.append(ctx.detect_track(d, c["interval"], 1, calc_angles=c["angles"], n_calls=N_CALLS))
        else:
            outs = new_outputs(torch, ctx.K, c["n"])      # fresh arrays: entries beyond a frame's count are never written
            ctx.detect_track(d, c["interval"], 1, calc_angles=c["angles"], n_calls=N_CALLS, outputs=outs)
            res.append(outs)
        if not pipelined:
            ctx.sync()
    ctx.sync()
    ctx.set_pipeline(False)
    return [r if c["host"] else host_copy(r) for c, r in zip(calls, res)]


def check_oracle(blob, c, got):
    """device outputs of call c == the oracle's detect, hand-off and 30 track() calls, frame by frame"""
    rects, counts, found, objs, _ = got
    angles = objs[:, 4:6].copy().view(np.float64)[:, 0]
    fr = frames(c)
    for f in range(c["n"]):
        want = oracle.detect(fr[f], blob, c["interval"], 1)
        n_det, fnd, obj = oracle.detect_track(fr[f], blob, c["interval"], 1, calc_angles=c["angles"], n_calls=N_CALLS)
        assert counts[f] == len(want) == n_det, f
        r = rects[f, :len(want)]
        nb = r[:, 5].copy().view(np.int32)[::2]
        assert [tuple(r[i, :5]) + (int(nb[i]),) for i in range(len(want))] == want, f
        assert found[f] == fnd, f
        if fnd:
            assert tuple(objs[f, :4]) == (obj["x"], obj["y"], obj["width"], obj["height"]), f
            assert abs(angles[f] - obj["angle"]) <= 1e-4, f


@pytest.mark.parametrize("memo", [False, True], ids=["strict", "memo"])
@pytest.mark.parametrize("name", list(SEQUENCES))
def test_pipelined_sequence_matches_unpipelined(blob, name, memo):
    import torch
    (mw, mh, mf), calls, with_oracle = SEQUENCES[name]
    ctx = Context(max_width=mw, max_height=mh, max_frames=mf, max_raw_per_frame=4096)
    try:
        ctx.set_track_memo(memo)
        dev = [torch.from_numpy(frames(c)).cuda() for c in calls]
        want = run(torch, ctx, calls, dev, pipelined=False)
        got = run(torch, ctx, calls, dev, pipelined=True)
    finally:
        ctx.close()
    for s, c in enumerate(calls):
        if c["host"]:
            assert got[s] == want[s], s
            assert any(got[s][1]), "the joining call must find faces"
        else:
            assert want[s][2].any(), (s, "the batches must contain faces")
            assert same_results(got[s], want[s]), (s, c)
    if with_oracle:
        for s in (0, len(calls) - 1):
            check_oracle(blob, calls[s], got[s])
