#!/usr/bin/env python
"""Per-frame device time of ht_tracker_step (headtrackr.Tracker lifecycle) against ht_stream_step_head on the same
streams: N 640x480 streams, device-resident frames and outputs, CUDA events around each step.

  tracker_wb      ht_tracker_step while every stream is in the whitebalance gate
  tracker_cs      ht_tracker_step in steady tracking (every stream in "CS")
  stream_head_cs  ht_stream_step_head in steady tracking

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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=10)
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
    line = json.dumps(res)
    print(line)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
