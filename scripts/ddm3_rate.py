"""Device time of the 3-D DynamicDistanceMap (ddm3d.cu) on the 30-cloud lidar scene (synth.make_clouds_3d), reach 0.5 m:

  bulk   every hit voxel (distinct Map::w2m of the 864 000 world points) added, then one update(), at 0.1 m and 0.05 m: update time,
         pops (update()'s processed count) and ns per pop;
  move   20 rounds of moving a 1 m box of obstacles through the 0.1 m map (remove the old position, add the new one, update()): the
         median time per update();
  query  distance(Vector3d, gradient) of the 864 000 world points on the 0.1 m map, in ms and points/s.

Device times are CUDA events (lama_dm3_kernel_times; the update time spans every brushfire launch of the call and the host's waits
between them), median of --reps runs after a warm-up, each bulk run on a fresh map.  The oracle's single-thread time on this host is
taken once per workload.  The card's name, power limit and max SM clock are read in the same call.  Prints one JSON line per
workload.  Needs a CUDA device.
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
import ddm3_oracle as T  # noqa: E402

CENTER = (0.0, 0.0, 1.5)
WINDOW = (8, 8, 6)   # the room (10 x 10 x 3 m) with the reach + 1 margin at 0.05 m
L2 = 0.5


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], text=True)
        return out.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def world_points():
    clouds, origins, quats = synth.make_clouds_3d(30)
    return np.concatenate([c @ synth.quat_matrix(q).T + o for c, o, q in zip(clouds, origins, quats)])


def hit_cells(res, pts):
    return np.unique(api.w2m3(res, pts), axis=0)


def bulk(res, cells, reps, oracle):
    ms, wall = [], []
    for r in range(reps + 1):
        g = api.DynamicDistanceMap3D(res, l2_max=L2, center=CENTER, window=WINDOW, timing=1)
        t0 = time.perf_counter()
        g.addObstacle(cells)
        pops = g.update()
        t1 = time.perf_counter()
        if r:
            ms.append(g.kernelTimes()[0]["update"])
            wall.append((t1 - t0) * 1e3)
    med = float(np.median(ms))
    out = dict(workload=f"dm3_bulk_{res}", obstacles=int(len(cells)), pops=int(pops), update_ms=med, update_ms_all=ms, wall_ms=float(np.median(wall)),
               ns_per_pop=med * 1e6 / pops, launches=g.runStats()["launches"], patches=g.bounds()[0])
    if oracle:
        o = T.Oracle(res, L2)
        t0 = time.perf_counter()
        o.addObstacle(cells)
        assert o.update() == pops
        out["oracle_s"] = time.perf_counter() - t0
        out["speedup_vs_oracle"] = out["oracle_s"] * 1e3 / med
    return out, g


def box_rounds(rounds=20):
    box = np.stack(np.meshgrid(*[np.arange(10)] * 3, indexing="ij"), -1).reshape(-1, 3).astype(np.uint32)
    at = np.array([T.OFFSET - 30, T.OFFSET - 20, T.OFFSET + 2], np.uint32)
    steps = []
    for r in range(rounds):
        nxt = at + np.array([3, 2, 0], np.uint32) if r % 4 != 3 else at - np.array([4, 1, 0], np.uint32)
        steps.append((box + at if r else None, box + nxt))
        at = nxt
    return steps


def move(g, cells, oracle):
    ms_ev, ms_wall, pops = [], [], []
    for gone, new in box_rounds():
        before = g.kernelTimes()[0]["update"]
        t0 = time.perf_counter()
        if gone is not None:
            g.removeObstacle(gone)
        g.addObstacle(new)
        pops.append(g.update())
        ms_wall.append((time.perf_counter() - t0) * 1e3)
        ms_ev.append(g.kernelTimes()[0]["update"] - before)
    out = dict(workload="dm3_box_move_0.1", rounds=len(ms_ev), update_ms=float(np.median(ms_ev)), wall_ms=float(np.median(ms_wall)),
               pops_median=int(np.median(pops)))
    if oracle:
        o = T.Oracle(0.1, L2)
        o.addObstacle(cells)
        o.update()
        ts = []
        for (gone, new), p in zip(box_rounds(), pops):
            t0 = time.perf_counter()
            if gone is not None:
                o.removeObstacle(gone)
            o.addObstacle(new)
            assert o.update() == p
            ts.append((time.perf_counter() - t0) * 1e3)
        out["oracle_ms"] = float(np.median(ts))
    return out


def query(g, pts, reps, oracle):
    ms = []
    for r in range(reps + 1):
        before = g.kernelTimes()[0]["distance"]
        d, grad = g.distance(pts)
        if r:
            ms.append(g.kernelTimes()[0]["distance"] - before)
    med = float(np.median(ms))
    out = dict(workload="dm3_query_0.1", points=int(len(pts)), distance_ms=med, points_per_s=len(pts) / (med * 1e-3))
    if oracle:
        o = T.Oracle(0.1, L2)
        o.addObstacle(hit_cells(0.1, pts))
        o.update()
        for gone, new in box_rounds():
            if gone is not None:
                o.removeObstacle(gone)
            o.addObstacle(new)
            o.update()
        t0 = time.perf_counter()
        do, go = o.distance(pts)
        out["oracle_ms"] = (time.perf_counter() - t0) * 1e3
        out["oracle_points_per_s"] = len(pts) / (out["oracle_ms"] * 1e-3)
        out["bit_equal"] = bool(np.array_equal(d, do) and np.array_equal(grad, go))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-oracle", action="store_true")
    a = ap.parse_args()
    if api.device_count() < 1:
        raise SystemExit("no CUDA device: the distance map rates are only measured on the GPU")
    gpu = card()
    pts = world_points()
    for res in (0.1, 0.05):
        cells = hit_cells(res, pts)
        r, g = bulk(res, cells, a.reps, not a.no_oracle)
        r["gpu"] = gpu
        print(json.dumps(r), flush=True)
        if res == 0.1:
            r = move(g, cells, not a.no_oracle)
            r["gpu"] = gpu
            print(json.dumps(r), flush=True)
            r = query(g, pts, a.reps, not a.no_oracle)
            r["gpu"] = gpu
            print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
