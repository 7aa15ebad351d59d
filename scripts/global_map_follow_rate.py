"""Rate of a following global-map render (FrequencyOccupancyMap(follow=True): Engine::render_scans in groups, the window moved between
them, the pool grown) on the device.

Set: the key scans of a GraphSlam2D run out and back along a 400 m x 16 m corridor (beams up to 10 m), rendered from scratch at 0.05 m
with free rays and at 0.1 m hits only, in a following map of dir_dim 16 (25.6 m / 51.2 m windows) and of dir_dim 64.  For each: device
time of the render kernels (CUDA events around each group's four kernels, summed), wall time of the whole call (it ends in a
synchronisation, so it includes the window shifts and pool growths), groups, shifts, parked entries, pool growths and the final pool,
median of warmed-up repeats on a fresh map each, and a cell-for-cell check against the oracle's render.  Prints one JSON line with the
card's name and power limit; writes it to OUT_DIR/global_map_follow_rate.json when given."""
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

REPEATS = 5


def _state(x, y, r):
    return [math.cos(r), math.sin(r), x, y]


def corridor_run(length=400.0, width=16.0, step=0.25, r_max=10.0, n_beams=360):
    segs = synth.make_corridor(length=length, width=width)
    xs = np.arange(0.0, length - 6.0, step)
    turn = np.linspace(0.0, np.pi, 10)[1:-1]
    path = [(x, 0.05 * np.sin(0.7 * x), 0.0) for x in xs] + [(xs[-1], 0.0, a) for a in turn]
    path += [(x, 0.05 * np.sin(0.7 * x), np.pi) for x in xs[::-1]]
    truth = np.array(path)
    angles = synth.beam_angles(n_beams, 360.0)
    rng_r, rng_o = np.random.default_rng(31), np.random.default_rng(32)
    g = api.GraphSlam2D()
    g.Init(*truth[0])
    cur = tuple(truth[0])
    for t in range(len(truth)):
        r = synth.cast(segs, truth[t], angles, 30.0) + rng_r.normal(0.0, 0.01, n_beams)
        p = synth.scan_points(r, angles)
        p = np.ascontiguousarray(p[np.hypot(p[:, 0], p[:, 1]) < r_max])
        if t:
            d = synth._between(tuple(truth[t - 1]), tuple(truth[t]))
            cur = synth._compose(cur, (d[0] + rng_o.normal(0, 0.01), d[1] + rng_o.normal(0, 0.01), d[2] + rng_o.normal(0, 0.005)))
        g.update(p, np.array(cur), float(t))
    cor, _, _ = g.keyPoses()
    return [g.keyCloud(i)[0] for i in range(len(cor))], [_state(*q) for q in cor], len(truth)


def measure(name, scans, states, res, full, dim):
    dev, wall, info = [], [], None
    for rep in range(REPEATS + 1):   # the first render also pays module loading
        m = api.FrequencyOccupancyMap(res, dir_dim=dim, follow=True, timing=1)
        t0 = time.perf_counter()
        cells = m.insertScans(scans, states, full=full)
        w_ms = (time.perf_counter() - t0) * 1e3
        kt, launches = m.kernelTimes()
        w = m.window()
        # render launches come four per group; shifts take two misc launches each, a pool growth one
        info = dict(cells=int(cells), groups=int(launches["raycast"]) // 4, shifts=w["shifts"], parked=w["parked"],
                    restored=w["restored"], pool_growths=int(launches["misc"]) - 2 * w["shifts"], pool=m.pool())
        if rep:
            dev.append(kt["raycast_ms"])
            wall.append(w_ms)
    o = gmo.OccupancyMap(res)
    co = o.insert_scans(scans, states, full)
    n, mn, mx = m.bounds()
    no, mn2, mx2 = o.bounds()
    same = n == no and (mn == mn2).all() and (mx == mx2).all() and co == info["cells"]
    if same:
        wd, h = int(mx[0] - mn[0]), int(mx[1] - mn[1])
        a, b = m.export(int(mn[0]), int(mn[1]), wd, h), o.export(int(mn[0]), int(mn[1]), wd, h)
        same = all((a[k] == b[k]).all() for k in ("occupied", "visited", "known"))
    return dict(set=name, dir_dim=dim, scans=len(scans), resolution=res, full=full, device_ms=float(np.median(dev)), device_ms_all=dev,
                wall_ms=float(np.median(wall)), wall_ms_all=wall, patches=int(n), cells_equal=bool(same), **info)


def main():
    out_dir = sys.argv[1] if len(sys.argv) > 1 else None
    if api.device_count() < 1:
        raise SystemExit("no CUDA device: the render rate is only measured on the GPU")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    keys, kst, n_scans = corridor_run()
    res = []
    for dim in (16, 64):
        res.append(measure("corridor_keys_full_0.05", keys, kst, 0.05, True, dim))
        res.append(measure("corridor_keys_hits_0.1", keys, kst, 0.1, False, dim))
    out = dict(card=card, scans=n_scans, key_poses=len(keys), results=res)
    line = json.dumps(out)
    print(line)
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "global_map_follow_rate.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
