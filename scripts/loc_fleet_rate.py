"""Rates of Loc2DFleet against stand-alone Loc2D handles on one shared map.

For R robots at B beams (R in 1, 16, 64, 256, 1024; B in 360, 1080): R robots spread along an 84 m corridor (the map read from the
oracle's file into a fixed dir_dim 64 window that holds it all, cov_blend 0, every update forced so that every robot tracks every
round).  One round = one Loc2DFleet.update of all R robots, or R Loc2D.update calls on R handles fed the same scans.  The two are
alternated round by round after WARMUP rounds of each; rounds/s and robot-updates/s come from the host clock around each round (every
round ends in a synchronisation).  After every timed pair the two sets of outputs (state, covariance, RMSE, solve counts) are compared
bit for bit.  Device memory: the drop in free device memory while each side's handles are created and their map read.

Prints one JSON line per (R, B) with the card's name and power limit; writes them to OUT_DIR/loc_fleet_rate.json when given."""
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from iris_lama_b200 import api, synth  # noqa: E402
from oracle import pyoracle as po  # noqa: E402
from test_gpu_window_follow import _out_and_back  # noqa: E402
from test_gpu_loc2d_follow import _cells  # noqa: E402

ROBOTS = (1, 16, 64, 256, 1024)
BEAMS = (360, 1080)
WARMUP, ROUNDS = 2, 10
OPTS = dict(dir_dim=64, center=(40.0, 0.0))


def free_bytes():
    import torch
    return torch.cuda.mem_get_info()[0]


def card():
    out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).splitlines()[0]
    name, limit = [s.strip() for s in out.split(",")]
    return name, limit


def run(path, data, R, B):
    truth, odom, scans = data
    T = len(scans)
    starts = [(k * 613) % (T - WARMUP - ROUNDS - 1) for k in range(R)]
    f0 = free_bytes()
    fleet = api.Loc2DFleet(api.Loc2DFleet.Options(**OPTS), R)
    fleet.distance_map.read(path)
    f1 = free_bytes()
    hs = []
    for _ in range(R):
        g = api.Loc2D(api.Loc2D.Options(**OPTS))
        g.distance_map.read(path)
        hs.append(g)
    f2 = free_bytes()
    for r, t in enumerate(starts):
        fleet.setPose(r, *truth[t])
        hs[r].setPose(*truth[t])
    robots = list(range(R))
    tf, ts, equal = 0.0, 0.0, True
    for i in range(WARMUP + ROUNDS):
        sc = [scans[starts[r] + i] for r in robots]
        od = [odom[starts[r] + i] for r in robots]
        t0 = time.perf_counter()
        fleet.update(robots, sc, od, force=[1] * R)
        t1 = time.perf_counter()
        for r in robots:
            hs[r].update(sc[r], od[r], force_update=True)
        t2 = time.perf_counter()
        if i >= WARMUP:
            tf += t1 - t0
            ts += t2 - t1
            st, cov, rmse, stats = fleet._get()
            for r in robots:
                g = hs[r]
                equal &= bool((st[r] == g.state()).all() and (cov[r] == g.getCovar()).all() and rmse[r] == g.getRMSE() and (stats[r] == g.solveStats()).all())
    beams = int(np.mean([s.shape[0] for s in scans]))
    return dict(robots=R, beams_per_scan_mean=beams, rounds=ROUNDS,
                fleet_rounds_per_s=ROUNDS / tf, fleet_robot_updates_per_s=ROUNDS * R / tf,
                single_rounds_per_s=ROUNDS / ts, single_robot_updates_per_s=ROUNDS * R / ts, speedup=ts / tf,
                fleet_device_mib=(f0 - f1) / 2**20, single_device_mib=(f1 - f2) / 2**20, bit_equal=equal, n_beams=B)


def main():
    name, limit = card()
    cells = _cells(synth.make_corridor(length=84.0))
    tmp = tempfile.mkdtemp()
    path = os.path.join(tmp, "corridor.sdm")
    od = po.DDM(0.05, 32, 1.0)
    od.add(cells)
    od.update()
    assert po.map_write("ddm", od, path)
    lines = []
    for B in BEAMS:
        data = _out_and_back(synth, n_beams=B, r_max=30.0)
        for R in ROBOTS:
            line = run(path, data, R, B)
            line.update(card=name, power_limit=limit)
            print(json.dumps(line), flush=True)
            lines.append(line)
    out = os.environ.get("OUT_DIR")
    if out:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "loc_fleet_rate.json"), "w") as fh:
            json.dump(lines, fh, indent=1)
    if not all(line["bit_equal"] for line in lines):
        sys.exit("fleet and stand-alone outputs differ")


if __name__ == "__main__":
    main()
