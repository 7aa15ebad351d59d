"""Device time of the coupled 3-D map update (OccupancyMap3D.updateMaps: om3d.cu's occupancy side and ddm3d.cu's segmented
brushfire) on the 30-cloud lidar scene (synth.make_clouds_3d), reach 0.5 m, at 0.1 m and 0.05 m, frequency maps:

  first        the 30 clouds into empty maps;
  incremental  the same 30 sensor poses again into those maps, with the scene's box moved 0.5 m in x and y.

Per case: CUDA-event times of the occupancy side (lama_om3_kernel_times[0]: records, sort, fold, filter, op list) and of the serial
side (lama_dm3_kernel_times[0]: every brushfire launch and the host's waits between them), the records (cell updates), the events
(setter calls that returned true), the pushes (events whose addObstacle / removeObstacle pushed a heap entry) and the pops (the sum
of the per-cloud update() counts).  The oracle composition (tests/emu/occ_dist3_oracle.cpp: every setter of the occupancy oracle that returns true
through the distance oracle, one host thread, which also reads each event's cell to count pushes) is timed on the same input and its results
checked equal.  One run per case after a warm-up at 0.1 m.  The card's name, power limit and max SM clock are read in the same call.
Prints one JSON line per case.  Needs a CUDA device.
"""
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
import test_occ_dist3d as T  # noqa: E402

CENTER = (0.0, 0.0, 1.5)
WINDOW = (8, 8, 6)
L2 = 0.5


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], text=True)
        return out.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def moved_clouds(origins, quats, shift=(0.5, 0.5, 0.0)):
    """the scene of make_clouds_3d with its box moved, cast from the same poses (same noise seed)"""
    scene = synth.make_scene_3d()
    scene["boxes"] = [(lo + np.array(shift), hi + np.array(shift)) for lo, hi in scene["boxes"]]
    dirs = synth.ring_lidar_dirs(32, 900)
    rng = np.random.Generator(np.random.PCG64(5))
    out = []
    for o, q in zip(origins, quats):
        r = synth.cast_3d(scene, o, dirs @ synth.quat_matrix(q).T, 30.0)
        out.append(dirs * (r + rng.normal(0.0, 0.005, size=r.shape))[:, None])
    return out


def run(res, batches, oracle=True):
    om = api.OccupancyMap3D(res, "frequency", center=CENTER, window=WINDOW, timing=1)
    dm = api.DynamicDistanceMap3D(res, l2_max=L2, center=CENTER, window=WINDOW, timing=1)
    o = T.OracleMaps(res, "frequency", None, l2_max=L2) if oracle else None
    rows = []
    for name, (clouds, origins, quats) in batches:
        om0, dm0 = om.kernelTimes()[0]["insert"], dm.kernelTimes()[0]["update"]
        t0 = time.perf_counter()
        cells, processed, counts = om.updateMaps(dm, clouds, origins, quats, counts=True)
        wall = time.perf_counter() - t0
        row = dict(case=name, resolution=res, max_sqdist=dm.max_sqdist, clouds=len(clouds), points=int(sum(len(c) for c in clouds)),
                   records=cells, events=counts["events"], pushes=counts["pushes"], pops=int(processed.sum()),
                   occupancy_ms=round(om.kernelTimes()[0]["insert"] - om0, 3), serial_ms=round(dm.kernelTimes()[0]["update"] - dm0, 3),
                   wall_ms=round(wall * 1e3, 3))
        if o is not None:
            t0 = time.perf_counter()
            n0, p0, c0 = o.updateMaps(clouds, origins, quats)
            row["oracle_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
            row["equal_to_oracle"] = bool(n0 == cells and c0 == counts and np.array_equal(p0, processed))
        rows.append(row)
    return rows


def main():
    clouds, origins, quats = synth.make_clouds_3d(30)
    moved = moved_clouds(origins, quats)
    gpu = card()
    run(0.1, [("warmup", (clouds[:3], origins[:3], quats[:3]))], oracle=False)
    for res in (0.1, 0.05):
        for row in run(res, [("first", (clouds, origins, quats)), ("incremental", (moved, origins, quats))]):
            row["gpu"] = gpu
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
