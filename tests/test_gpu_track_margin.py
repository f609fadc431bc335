"""GPU parity of k_track on frames built to sit near a truncation boundary (tests/test_track_margin_host.py).

On a trap frame the exact value of l1 (or of the first shift) lies within a few 1e-7 of an integer, and the
reference's serial sums truncate it on the other side.  k_track's parallel sums are far closer to exact, so from them
alone the kernel would truncate the other way: it must see that the value is within its tolerance of the integer and
take moments_serial.  So on every trap launch serial_passes >= 1, whatever the rounding, and every output equals the
oracle's - at canvas sizes up to 3840x2160 (each test makes its own Context: the session one stops at 1280x720), over
the cluster sizes, thread counts, the window memo and a launch of 256 streams that engages the longest-chain-first
tiers.
"""
import math

import pytest

import oracle
from test_track_margin_host import CONTROLS, FAMILIES, SHIFT_FAMILIES, find_trap

pytestmark = pytest.mark.gpu

N_CALLS = 3
_WANT = {}


def oracle_calls(t):
    """The oracle's N_CALLS track() calls of a trap: [(x, y, width, height, angle, search window)]."""
    if t["name"] not in _WANT:
        ot = oracle.CamshiftTracker(calc_angles=t["calc"])
        ot.init_tracker(t["A"], *t["rect"])
        out = []
        for _ in range(N_CALLS):
            ot.track(t["B"])
            o = ot.track_obj()
            out.append((o["x"], o["y"], o["width"], o["height"], o["angle"], ot.search_window()))
        _WANT[t["name"]] = out
    return _WANT[t["name"]]


def assert_call(obj, win, want, what):
    assert (obj["x"], obj["y"], obj["width"], obj["height"]) == want[:4], what
    # a window without mass gives NaN moments and a NaN angle, in the reference as in the kernel
    assert abs(obj["angle"] - want[4]) <= 1e-4 or (math.isnan(obj["angle"]) and math.isnan(want[4])), what
    assert win == want[5], what


CONFIGS = {
    "default": {},
    "cluster1": {"HT_TRACK_CLUSTER": "1"},
    "cluster2": {"HT_TRACK_CLUSTER": "2"},
    "cluster4": {"HT_TRACK_CLUSTER": "4"},
    "cluster8": {"HT_TRACK_CLUSTER": "8"},
    "cluster16": {"HT_TRACK_CLUSTER": "16"},
    "nt128": {"HT_TRACK_NT": "128"},
    "nt512": {"HT_TRACK_NT": "512"},
    "nomemo": {"HT_TRACK_MEMO": "0"},
}


@pytest.mark.parametrize("config", list(CONFIGS))
@pytest.mark.parametrize("name", list(FAMILIES) + list(SHIFT_FAMILIES) + list(CONTROLS))
def test_trap_frames_match_oracle(name, config, monkeypatch):
    from headtrackr_b200 import Context
    for k, v in CONFIGS[config].items():
        monkeypatch.setenv(k, v)
    t = find_trap(name)
    want = oracle_calls(t)
    H, W = t["B"].shape[:2]
    c = Context(max_width=W, max_height=H, max_frames=1)
    try:
        c.track_init(t["A"], [t["rect"]], calc_angles=t["calc"])
        c.debug_track_stats(reset=True)
        for call in range(N_CALLS):
            objs, wins = c.track(t["B"])
            assert_call(objs[0], wins[0], want[call], (name, config, call))
            if call == 0 and not t["control"]:
                st = c.debug_track_stats(reset=True)
                assert st["serial_passes"] >= 1, st
    finally:
        c.close()


def test_trap_frames_in_a_tiered_launch():
    """256 streams of the 2560x1440 trap, built on the device: the launch orders them longest-chain-first and runs
    them in tiers (clusters of 8, 4 and 2).  Every stream equals the oracle, and every stream takes the fallback."""
    import torch
    from headtrackr_b200 import Context
    t = find_trap("1440p")
    want = oracle_calls(t)
    H, W = t["B"].shape[:2]
    N, chunk = 256, 16
    c = Context(max_width=W, max_height=H, max_frames=N)
    try:
        A = torch.from_numpy(t["A"]).cuda().unsqueeze(0).expand(chunk, H, W, 4).contiguous()
        for s0 in range(0, N, chunk):
            c.track_init(A, [t["rect"]] * chunk, slots=list(range(s0, s0 + chunk)), calc_angles=t["calc"])
        del A
        B = torch.from_numpy(t["B"]).cuda().unsqueeze(0).expand(N, H, W, 4).contiguous()
        c.debug_track_stats(reset=True)
        for call in range(N_CALLS):
            objs, wins = c.track(B)
            for i in range(N):
                assert_call(objs[i], wins[i], want[call], (i, call))
            if call == 0:
                st = c.debug_track_stats(reset=True)
                assert st["serial_passes"] >= N, st
    finally:
        c.close()
