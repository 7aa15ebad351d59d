"""Device time of the truncated signed distance map (tsdm.cu): fusing all 5 000 config-4 scans in 2-D, a 3-D lidar set, and toMesh.

CUDA events (lama_tsdm_kernel_times), median of --reps timed runs after one warm-up run, each on a fresh map.  Records are the
fold records (walked voxels that are not skipped); the algorithmic bytes count 16 B of cell state per record (an 8-byte cell read and
written), against the H100 SXM's 3.35 TB/s.  The oracle's single-thread time on the host is taken once per workload.  Prints one JSON
line per workload.  Needs a CUDA device.
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
import tsdm_oracle as T  # noqa: E402


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], text=True)
        return out.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def measure(name, clouds, origins, quats, res, is3d, reps, oracle):
    ms_fuse, ms_mesh = [], []
    for r in range(reps + 1):
        g = api.TruncatedSignedDistanceMap(res, is3d=is3d, center=(0, 0, 1.5) if is3d else (0, 0, 0), timing=1)
        g.insertPointClouds(clouds, origins, quats)
        v, _ = g.toMesh()
        ms, _ = g.kernelTimes()
        if r:
            ms_fuse.append(ms["insert"])
            ms_mesh.append(ms["mesh"])
    n_pts = sum(len(c) for c in clouds)
    out = dict(workload=name, clouds=len(clouds), points=n_pts, fuse_ms=float(np.median(ms_fuse)), mesh_ms=float(np.median(ms_mesh)),
               mesh_vertices=int(len(v)), patches=g.bounds()[0])
    if oracle:
        o = T.Oracle(res, is3d)
        t0 = time.perf_counter()
        o.insertPointClouds(clouds, origins, quats)
        out["oracle_fuse_s"] = time.perf_counter() - t0
        t0 = time.perf_counter()
        o.toMesh()
        out["oracle_mesh_s"] = time.perf_counter() - t0
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-oracle", action="store_true")
    a = ap.parse_args()
    if api.device_count() < 1:
        raise SystemExit("no CUDA device: the fusion rate is only measured on the GPU")
    gpu = card()
    ds = synth.make_dataset("loop", 5000)
    org = np.c_[ds.truth[:, :2], np.zeros(len(ds.truth))]
    q = np.array([[0, 0, np.sin(t / 2), np.cos(t / 2)] for t in ds.truth[:, 2]])
    c3, o3, q3 = synth.make_clouds_3d(30)
    for args in (("config4_2d_0.05", list(ds.scans), org, q, 0.05, False), ("lidar3d_30_0.05", c3, o3, q3, 0.05, True),
                 ("lidar3d_30_0.1", c3, o3, q3, 0.1, True)):
        r = measure(*args, a.reps, not a.no_oracle)
        r["gpu"] = gpu
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
