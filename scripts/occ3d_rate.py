"""Device time of the 3-D occupancy maps (om3d.cu): 30 clouds of the 32-ring lidar (864 000 points) inserted with full rays, both
kinds, at 0.05 m and 0.1 m.

CUDA events (lama_om3_kernel_times), median of --reps timed runs after one warm-up run, each on a fresh map.  C = the cell updates
(hits and ray cells); the algorithmic bytes count 8 B per update (a 4-byte cell read and written), against the H100 SXM's 3.35 TB/s.
The oracle's single-thread time on the host is taken once per workload.  The card's name, power limit and max SM clock are read in
the same call.  Prints one JSON line per workload.  Needs a CUDA device.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from iris_lama_b200 import api, synth  # noqa: E402
import occ3d_oracle as T  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], text=True)
        return out.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def measure(clouds, origins, quats, res, kind, reps, oracle):
    ms = []
    for r in range(reps + 1):
        g = api.OccupancyMap3D(res, kind, center=(0, 0, 1.5), timing=1)
        cells = g.insertPointClouds(clouds, origins, quats, full=True)
        t, launches = g.kernelTimes()
        if r:
            ms.append(t["insert"])
    med = float(np.median(ms))
    out = dict(workload=f"lidar3d_30_{res}_{kind}", clouds=len(clouds), points=int(sum(len(c) for c in clouds)), cell_updates=int(cells),
               insert_ms=med, insert_ms_all=ms, launches=int(launches["insert"]), patches=g.bounds()[0],
               updates_per_s=cells / (med * 1e-3), bytes_share_of_hbm=(8.0 * cells / (med * 1e-3)) / HBM_BYTES_PER_S)
    if oracle:
        o = T.Oracle(res, kind)
        t0 = time.perf_counter()
        o.insertPointClouds(clouds, origins, quats, full=True)
        out["oracle_insert_s"] = time.perf_counter() - t0
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-oracle", action="store_true")
    a = ap.parse_args()
    if api.device_count() < 1:
        raise SystemExit("no CUDA device: the insertion rate is only measured on the GPU")
    gpu = card()
    c3, o3, q3 = synth.make_clouds_3d(30)
    for res in (0.05, 0.1):
        for kind in ("frequency", "logodds"):
            r = measure(c3, o3, q3, res, kind, a.reps, not a.no_oracle)
            r["gpu"] = gpu
            print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
