#!/usr/bin/env python
"""CPU model of k_cascade's shared-memory LOAD WAVEFRONTS (the resource that bounds the kernel, DESIGN.md §5.1).

For one synthetic frame it evaluates the cascade for every window with numpy (same arithmetic and order as the
reference; checked against the oracle's survivor count), then replays the kernel's work distribution tile by tile —
dense first group, 32 bank-class survivor lists, lane-per-window stage groups, warp-per-window late stages — and
counts the LDS wavefronts each variant would issue, including bank-conflict replays.  Used to rank layout /
grouping ideas before spending GPU time on them.  Its counts depend on the kernel's layout, not on the GPU; check
the `current` variant against an ncu capture of k_cascade (shared-load wavefronts and conflict replays per frame)
before relying on it.

    python tools/cascade_wavefront_model.py [frame_index] [W H]
"""
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import oracle  # noqa: E402  (test infrastructure; this is an analysis tool, not the product)
from headtrackr_b200 import synth  # noqa: E402

TW, TH = 32, 16
TILE_ROWS = 4 * TH + 22


def stage_tables(c):
    """per stage: list of features as (p points, n points, a_fail, a_pass), distinct points, threshold"""
    out = []
    for (count, first, thr) in c["stages"]:
        feats, pts = [], []
        for k in range(first, first + count):
            f = c["features"][k]
            pp = list(dict.fromkeys(p for p in f["p"][: f["size"]] if p[0] >= 0))
            nn = list(dict.fromkeys(p for p in f["n"][: f["size"]] if p[0] >= 0))
            feats.append((pp, nn, f["a_fail"], f["a_pass"]))
            pts += pp + nn
        out.append(dict(feats=feats, points=list(dict.fromkeys(pts)), refs=len(pts), thr=thr))
    return out


def window_depths(frame, blob, interval=5):
    """-> list per scale of (qw, qh, depth[4, qh, qw]) where depth = number of stages passed (n_stages = detection)"""
    c = synth.parse_blob(blob)
    st = stage_tables(c)
    pyr = oracle.Pyramid(oracle.grayscale(frame), interval)
    g = pyr.geom
    nxt = g.next
    scales = []
    for i in range(g.scale_upto):
        qw, qh = g.w[i + 2 * nxt] - c["width"] // 4, g.h[i + 2 * nxt] - c["height"] // 4
        if qw <= 0 or qh <= 0:
            continue
        pad = 32

        def padded(a):
            return np.pad(a, ((0, pad), (0, pad)))
        p0, p1 = padded(pyr.plane(i)), padded(pyr.plane(i + nxt))
        p2 = [padded(pyr.plane(i + 2 * nxt, q)) for q in range(4)]
        depth = np.zeros((4, qh, qw), np.int32)
        for q in range(4):
            dx, dy = q & 1, q >> 1
            gy, gx = np.mgrid[0:qh, 0:qw]
            gy, gx = gy.ravel(), gx.ravel()
            alive = np.arange(gx.size)
            for j, s in enumerate(st):
                if alive.size == 0:
                    break
                ax, ay = gx[alive], gy[alive]

                def px(pt):
                    z, x, y = pt
                    if z == 0:
                        return p0[4 * ay + 2 * dy + y, 4 * ax + 2 * dx + x]
                    if z == 1:
                        return p1[2 * ay + dy + y, 2 * ax + dx + x]
                    return p2[q][ay + y, ax + x]
                total = np.zeros(alive.size)
                for (pp, nn, a_fail, a_pass) in s["feats"]:
                    pm = np.minimum.reduce([px(p) for p in pp])
                    nm = np.maximum.reduce([px(p) for p in nn])
                    total = total + np.where(pm > nm, a_pass, a_fail)
                ok = ~(total < s["thr"])
                alive = alive[ok]
                depth[q].ravel()[alive] = j + 1
        scales.append((qw, qh, depth))
    return st, scales


def expanded_offset(pt, TP):
    z, x, y = pt
    region = TILE_ROWS * TP
    return y * TP + x if z == 0 else (region + TP + 2 * x + 2 * y * TP if z == 1 else region + 4 * x + 4 * y * TP)


class Variant:
    def __init__(self, name, groups, late_first=8, TP=160, dx_copy=False, dx_lists=False):
        self.name, self.groups, self.late_first, self.TP = name, groups, late_first, TP
        self.dx_copy, self.dx_lists = dx_copy, dx_lists


def simulate(st, scales, v):
    TP = v.TP
    offs = [np.array([expanded_offset(p, TP) for p in s["points"]]) for s in st]
    n_loads = [len(o) for o in offs]
    tot = dict(dense=0, lists=0, conflicts=0, late=0, overhead=0, iters=0)
    n_tiles = 0
    for (qw, qh, depth) in scales:
        for ty in range((qh + TH - 1) // TH):
            for tx in range((qw + TW - 1) // TW):
                n_tiles += 1
                # windows of the tile: arrays lx, ly, q, depth
                ys = np.arange(ty * TH, min(qh, ty * TH + TH))
                xs = np.arange(tx * TW, min(qw, tx * TW + TW))
                d = depth[:, ys[:, None], xs[None, :]]                       # [4, ny, nx]
                qq, ly, lx = np.meshgrid(np.arange(4), ys - ty * TH, xs - tx * TW, indexing="ij")
                qq, ly, lx, d = qq.ravel(), ly.ravel(), lx.ravel(), d.ravel()
                first = True
                alive_mask = np.ones(d.size, bool)
                for grp in v.groups:
                    if first:
                        # dense: warp-iteration = (q, ly): 32 lanes lx; later stages of the group run per iteration if any lane alive
                        key = qq * TH + ly
                        for si, j in enumerate(grp):
                            if si == 0:
                                tot["dense"] += len(np.unique(key)) * n_loads[j]
                            else:
                                live = alive_mask & (d >= j)
                                tot["dense"] += len(np.unique(key[live])) * n_loads[j]
                        first = False
                    else:
                        idx = np.nonzero(alive_mask)[0]
                        if idx.size == 0:
                            break
                        dxs, dys = qq[idx] & 1, qq[idx] >> 1
                        a0 = (4 * lx[idx] + 2 * dxs) + (4 * ly[idx] + 2 * dys) * TP
                        cls = (a0 >> 2) & 31
                        if v.dx_copy:
                            cls = (((4 * lx[idx]) + (4 * ly[idx] + 2 * dys) * TP) >> 2) & 31
                        # per-class lists in compaction order (index order is close enough)
                        order = np.argsort(cls, kind="stable")
                        idx, cls, dxs, a0 = idx[order], cls[order], dxs[order], a0[order]
                        counts = np.bincount(cls, minlength=32)
                        start = np.concatenate([[0], np.cumsum(counts)[:-1]])
                        pos = np.arange(idx.size) - start[cls]                    # entry index inside its class list
                        if v.dx_lists:   # entries of dx = 0 first, then dx = 1, aligned over the classes
                            c0 = np.bincount(cls[dxs == 0], minlength=32)
                            c1 = np.bincount(cls[dxs == 1], minlength=32)
                            m0 = c0.max() if c0.size else 0
                            o2 = np.lexsort((dxs, cls))
                            idx, cls, dxs, a0 = idx[o2], cls[o2], dxs[o2], a0[o2]
                            start0 = np.concatenate([[0], np.cumsum(np.bincount(cls, minlength=32))[:-1]])
                            p_in = np.arange(idx.size) - start0[cls]
                            pos = np.where(dxs == 0, p_in, m0 + p_in - c0[cls])
                            n_iter = m0 + (c1.max() if c1.size else 0)
                        else:
                            n_iter = counts.max()
                        tot["iters"] += n_iter
                        tot["overhead"] += n_iter                             # the list read itself (LDS.U16 per iteration)
                        for si, j in enumerate(grp):
                            live = d[idx] >= j if si > 0 else np.ones(idx.size, bool)
                            its = np.unique(pos[live])
                            tot["lists"] += len(its) * n_loads[j]
                            if not v.dx_copy and not v.dx_lists:
                                # conflict replay: class k (dx = 1) next to class k+1 (dx = 0) in the same iteration, for
                                # offsets with bit 1 set, unless both lanes read the very same word
                                n_c = int(((offs[j] & 3) >= 2).sum())
                                word_base = (a0 >> 2)
                                for e in its:
                                    m = live & (pos == e)
                                    k1 = {int(c): (int(w), int(x)) for c, w, x in zip(cls[m], word_base[m], dxs[m])}
                                    hit = False
                                    for c, (w, x) in k1.items():
                                        if x == 1:
                                            nb = k1.get((c + 1) & 31)
                                            if nb is not None and nb[1] == 0 and nb[0] != w + 1:
                                                hit = True
                                                break
                                    if hit:
                                        tot["conflicts"] += n_c
                    # survivors of the group
                    alive_mask &= d >= (grp[-1] + 1)
                    tot["overhead"] += 2 * 64                                   # compaction: raw reads + count reads
                # late stages: one warp per window, a feature per lane, ~10 predicated byte loads per chunk of 32 features
                idx = np.nonzero(alive_mask)[0]
                for w in idx:
                    a0 = (4 * lx[w] + 2 * (qq[w] & 1)) + (4 * ly[w] + 2 * (qq[w] >> 1)) * TP
                    for j in range(v.late_first, len(st)):
                        if d[w] < j:
                            break
                        feats = st[j]["feats"]
                        for base in range(0, len(feats), 32):
                            chunk = feats[base:base + 32]
                            for slot in range(5):
                                for which in (0, 1):
                                    addrs = [a0 + expanded_offset(f[which][slot], TP) for f in chunk if len(f[which]) > slot]
                                    if not addrs:
                                        continue
                                    words = np.unique(np.array(addrs) >> 2)
                                    tot["late"] += int(np.bincount(words & 31, minlength=32).max())
    tot["tiles"] = n_tiles
    tot["total"] = tot["dense"] + tot["lists"] + tot["conflicts"] + tot["late"] + tot["overhead"]
    return tot


def simulate_quad(st, scales, groups, late_first=8, loads_per_point=1.75):
    """What-if: phase-planar tile (level 0 in 4 planes by x mod 4, level 1 in 2, level 2 as is) where a LANE evaluates
    the 4 x-adjacent windows (same ly, same phase) from 32-bit loads: a point costs 1 aligned or 2 unaligned LDS.32
    per lane (1.75 on average) and serves 4 windows.  A quad stays in the lists while any of its windows is alive."""
    n_loads = [len(s["points"]) * loads_per_point for s in st]
    tot = dict(dense=0.0, lists=0.0, conflicts=0, late=0, overhead=0, iters=0)
    n_tiles = 0
    for (qw, qh, depth) in scales:
        for ty in range((qh + TH - 1) // TH):
            for tx in range((qw + TW - 1) // TW):
                n_tiles += 1
                ys = np.arange(ty * TH, min(qh, ty * TH + TH))
                xs = np.arange(tx * TW, min(qw, tx * TW + TW))
                d = np.zeros((4, TH, TW), np.int32) - 1
                d[:, : len(ys), : len(xs)] = depth[:, ys[:, None], xs[None, :]]
                dq = d.reshape(4, TH, TW // 4, 4).max(axis=3)                 # depth of a quad = its deepest window
                qq, ly, g = np.meshgrid(np.arange(4), np.arange(TH), np.arange(TW // 4), indexing="ij")
                qq, ly, g, dq = qq.ravel(), ly.ravel(), g.ravel(), dq.ravel()
                valid = dq >= 0
                alive = valid.copy()
                first = True
                for grp in groups:
                    if first:
                        key = (qq * TH + ly) // 4                              # a warp iteration = 4 rows x 8 quads
                        for si, j in enumerate(grp):
                            live = alive & (dq >= j) if si > 0 else alive
                            tot["dense"] += len(np.unique(key[live])) * n_loads[j]
                        first = False
                    else:
                        idx = np.nonzero(alive)[0]
                        if idx.size == 0:
                            break
                        cls = (g[idx] + 8 * (ly[idx] & 3)) & 31                # bank of the quad's base word (pitch = 8 words mod 32)
                        counts = np.bincount(cls, minlength=32)
                        n_iter = counts.max()
                        order = np.argsort(cls, kind="stable")
                        idx, cls = idx[order], cls[order]
                        start = np.concatenate([[0], np.cumsum(counts)[:-1]])
                        pos = np.arange(idx.size) - start[cls]
                        tot["iters"] += n_iter
                        tot["overhead"] += n_iter
                        for si, j in enumerate(grp):
                            live = dq[idx] >= j if si > 0 else np.ones(idx.size, bool)
                            tot["lists"] += len(np.unique(pos[live])) * n_loads[j]
                    alive &= dq >= (grp[-1] + 1)
                    tot["overhead"] += 2 * 16
        # late stages: as in the current design (taken from the byte-layout model by the caller)
    tot["tiles"] = n_tiles
    return tot


def main():
    idx = int(sys.argv[1]) if len(sys.argv) > 1 else 0
    W, H = (int(sys.argv[2]), int(sys.argv[3])) if len(sys.argv) > 3 else (640, 480)
    blob = synth.load_cascade_blob()
    frame = synth.frame(idx, W, H)
    st, scales = window_depths(frame, blob)
    n_det = sum(int((d == len(st)).sum()) for (_, _, d) in scales)
    n_win = sum(d.size for (_, _, d) in scales)
    raw, stats = oracle.Pyramid(oracle.grayscale(frame)).cascade_raw(blob)
    assert n_win == stats.windows and n_det == stats.n_raw, (n_win, stats.windows, n_det, stats.n_raw)
    print(f"frame {idx} {W}x{H}: {n_win} windows, {n_det} raw detections (== oracle)")
    print("distinct loads per stage:", [len(s["points"]) for s in st])
    variants = [
        Variant("current {0,1}{2}{3}{4,5}{6,7} late>=8", [[0, 1], [2], [3], [4, 5], [6, 7]]),
        Variant("round-1a {0,1}{2,3}{4,5}{6,7}", [[0, 1], [2, 3], [4, 5], [6, 7]]),
        Variant("all single {0}{1}{2}{3}{4,5}{6,7}", [[0], [1], [2], [3], [4, 5], [6, 7]]),
        Variant("x-phase-separated lists", [[0, 1], [2], [3], [4, 5], [6, 7]], dx_lists=True),
        Variant("dx = 1 windows on a tile copy shifted by 2 B", [[0, 1], [2], [3], [4, 5], [6, 7]], dx_copy=True),
        Variant("pitch 164", [[0, 1], [2], [3], [4, 5], [6, 7]], TP=164),
        Variant("lane-per-window up to stage 9", [[0, 1], [2], [3], [4, 5], [6, 7], [8, 9]], late_first=10),
    ]
    print(f"{'variant':52s} {'total':>9s} {'dense':>8s} {'lists':>8s} {'confl':>8s} {'late':>8s} {'ovh':>7s} {'iters':>7s}  per tile")
    late_now = None
    for v in variants:
        t = simulate(st, scales, v)
        if late_now is None:
            late_now = t["late"]
        print(f"{v.name:52s} {t['total']:9d} {t['dense']:8d} {t['lists']:8d} {t['conflicts']:8d} {t['late']:8d} "
              f"{t['overhead']:7d} {t['iters']:7d}  {t['total'] / t['tiles']:.0f}")
    for name, groups in (("QUAD lanes {0,1}{2}{3}{4,5}{6,7}", [[0, 1], [2], [3], [4, 5], [6, 7]]),
                         ("QUAD lanes {0,1}{2,3}{4,5}{6,7}", [[0, 1], [2, 3], [4, 5], [6, 7]])):
        t = simulate_quad(st, scales, groups)
        total = t["dense"] + t["lists"] + late_now + t["overhead"]
        print(f"{name:52s} {int(total):9d} {int(t['dense']):8d} {int(t['lists']):8d} {0:8d} {late_now:8d} "
              f"{t['overhead']:7d} {t['iters']:7d}  {total / t['tiles']:.0f}")


if __name__ == "__main__":
    main()
