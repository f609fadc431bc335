#!/usr/bin/env python
"""DRAM bytes of one captured kernel launch -> build/cascade_dram.json (bench.py's roofline.traffic; git-ignored).

    python tools/ncu_dram.py cascade.ncu-rep --frames 32 --width 640 --height 480

`--frames` is the number of frames the captured launch covered (one L2 wave of the profile run).  The value is
dram__bytes_read.sum + dram__bytes_write.sum of that launch divided by its frames; bench.py scales it to its own
launch size and reports the file name as the source.
"""
import argparse
import csv
import json
import subprocess
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent


def raw_page(rep):
    out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    hdr, units = rows[0], rows[1]
    return [dict(zip(hdr, r)) for r in rows[2:]], dict(zip(hdr, units))


def to_bytes(v, unit):
    x = float(v.replace(",", ""))
    return x * {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(unit, 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("rep")
    ap.add_argument("--frames", type=int, required=True)
    ap.add_argument("--width", type=int, default=640)
    ap.add_argument("--height", type=int, default=480)
    ap.add_argument("--out", default=str(ROOT / "build" / "cascade_dram.json"))
    a = ap.parse_args()
    rows, units = raw_page(a.rep)
    r = rows[0]
    rd = to_bytes(r["dram__bytes_read.sum"], units["dram__bytes_read.sum"])
    wr = to_bytes(r["dram__bytes_write.sum"], units["dram__bytes_write.sum"])
    d = {"kernel": r.get("Kernel Name", "k_cascade"), "width": a.width, "height": a.height, "frames_in_launch": a.frames,
         "dram_bytes_read": rd, "dram_bytes_write": wr, "dram_bytes_per_frame": (rd + wr) / a.frames,
         "algorithmic_bytes_per_frame": a.width * a.height * 4,
         "source": f"{Path(a.out).name} <- ncu --set full capture {Path(a.rep).name}"}
    Path(a.out).parent.mkdir(parents=True, exist_ok=True)
    Path(a.out).write_text(json.dumps(d, indent=1) + "\n")
    print(json.dumps(d))


if __name__ == "__main__":
    main()
