#!/usr/bin/env python
"""k_group's device time on crowded frames (ht_profile, class "group"), next to the rest of detection.

One warp groups one frame with O(n^2) lane loops, so its cost grows with the square of the raw list: a 640x480
synth.crowd_frame has about 1,900 raw windows and 330 groups, bench.py's frames a few dozen windows.  This runs
ht_detect on N crowded frames (a few distinct crowds repeated, device-resident) with max_raw_per_frame 4096 and prints
one JSON line with the median per-call time of each kernel class over the timed repeats.

    python tools/profile_group_crowd.py [--frames 1024] [--repeats 5] [--min-neighbors 1]
"""
import argparse
import json
import statistics
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from headtrackr_b200 import Context, synth  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1024)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--width", type=int, default=640)
    ap.add_argument("--height", type=int, default=480)
    ap.add_argument("--min-neighbors", type=int, default=1)
    a = ap.parse_args()
    import torch
    W, H, n = a.width, a.height, a.frames
    uniq = np.stack([synth.crowd_frame(s, W, H, side=28, pitch=30, jitter=2) for s in range(4)])
    dev = torch.from_numpy(uniq).cuda()[torch.arange(n, device="cuda") % len(uniq)].contiguous()
    c = Context(max_width=W, max_height=H, max_frames=n, max_raw_per_frame=4096)
    try:
        c.detect(dev[:8], 5, a.min_neighbors)                 # plan, arena, cascade upload
        raw = [c.debug_raw(i)[1] for i in range(len(uniq))]
        per = {}
        for _ in range(a.repeats):
            c.profile(True)
            c.detect(dev, 5, a.min_neighbors)
            for k, (ms, _) in c.profile_read(reset=True).items():
                per.setdefault(k, []).append(ms)
            c.profile(False)
        out = dict(frames=n, width=W, height=H, min_neighbors=a.min_neighbors, raw_per_frame=raw,
                   warning=c.last_warning, gpu=torch.cuda.get_device_name(0),
                   ms={k: round(statistics.median(v), 3) for k, v in per.items() if max(v) > 0})
        print(json.dumps(out))
    finally:
        c.close()


if __name__ == "__main__":
    main()
