"""Rate of the global-map render (k_render_scans: GraphSlam2D::generateOccupancyMap from scratch) on the device.

Sets: the key scans of a GraphSlam2D run over the two-lap loop world (synth "loop", 1600 scans, 1080 beams) at their corrected poses,
rendered at 0.05 m with free rays and at 0.1 m hits only (the two maps generateOccupancyMap(full) makes); every 10th scan and all scans
of the 5 000-scan config-4 trajectory at their true poses, 0.05 m with free rays.  For each: device time of the render (CUDA events
around its four kernels, median of warmed-up repeats on a fresh map each), cell updates C, algorithmic bytes C * 8 (SURVEY 8(d)) over
that time as a share of the H100 SXM's 3.35 TB/s, the CPU oracle's single-thread time of the
same render on the same host, and a cell-for-cell check of the device map against the oracle's.  Prints one JSON line with the card's
name and power limit; writes it to OUT_DIR/global_map_rate.json when given."""
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from iris_lama_b200 import api, synth  # noqa: E402
import global_map_oracle as gmo  # noqa: E402

PEAK = 3.35e12
REPEATS = 5


def _state(x, y, r):
    return [math.cos(r), math.sin(r), x, y]


def measure(name, scans, states, res, full):
    times, cells = [], 0
    for rep in range(REPEATS + 1):   # the first render also pays module loading and allocation
        m = api.FrequencyOccupancyMap(res, timing=1)
        cells = m.insertScans(scans, states, full=full)
        ms = m.kernelTimes()[0]["raycast_ms"]
        if rep:
            times.append(ms)
    ms = float(np.median(times))
    o = gmo.OccupancyMap(res)
    t0 = time.perf_counter()
    co = o.insert_scans(scans, states, full)
    oracle_s = time.perf_counter() - t0
    n, mn, mx = m.bounds()
    no, mn2, mx2 = o.bounds()
    same = n == no and (mn == mn2).all() and (mx == mx2).all() and co == cells
    if same:
        w, h = int(mx[0] - mn[0]), int(mx[1] - mn[1])
        a, b = m.export(int(mn[0]), int(mn[1]), w, h), o.export(int(mn[0]), int(mn[1]), w, h)
        same = all((a[k] == b[k]).all() for k in ("occupied", "visited", "known"))
    beams = int(sum(len(s) for s in scans))
    return dict(set=name, scans=len(scans), beams=beams, resolution=res, full=full, cells=int(cells), device_ms=ms, device_ms_all=times,
                cells_per_s=cells / (ms * 1e-3), bytes=8 * int(cells), share_of_peak_bw=8 * cells / (ms * 1e-3) / PEAK, oracle_s=oracle_s,
                speedup_vs_oracle=oracle_s / (ms * 1e-3), patches=int(n), cells_equal=bool(same))


def main():
    out_dir = sys.argv[1] if len(sys.argv) > 1 else None
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    if api.device_count() < 1:
        raise SystemExit("no CUDA device: the render rate is only measured on the GPU")
    res = []
    ds = synth.make_dataset("loop", 1600, n_beams=1080)
    g = api.GraphSlam2D()
    g.Init(*ds.truth[0])
    for t in range(ds.n_scans):
        g.update(ds.scans[t], ds.odom[t], float(t))
    cor, _, _ = g.keyPoses()
    keys = [g.keyCloud(i)[0] for i in range(len(cor))]
    kst = [_state(*p) for p in cor]
    res.append(measure("graph_keys_full_0.05", keys, kst, 0.05, True))
    res.append(measure("graph_keys_hits_0.1", keys, kst, 0.1, False))
    big = synth.make_dataset("loop", 5000)
    tst = [_state(*p) for p in big.truth]
    res.append(measure("config4_every10th_full_0.05", big.scans[::10], tst[::10], 0.05, True))
    res.append(measure("config4_all_full_0.05", big.scans, tst, 0.05, True))
    out = dict(card=card, key_poses=len(cor), results=res)
    line = json.dumps(out)
    print(line)
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "global_map_rate.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
