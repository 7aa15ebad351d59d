"""Every CUDA buffer, event and stream of the host code is owned through csrc/cuda_owned.h: no other source allocates or releases one
directly, the header stands on its own, and creating and destroying every handle kind leaves the process's device memory where it was."""
import json
import os
import pathlib
import re
import shutil
import subprocess
import sys
import textwrap

import pytest

ROOT = pathlib.Path(__file__).resolve().parents[1]
CSRC = ROOT / "iris_lama_b200" / "csrc"
HEADER = CSRC / "cuda_owned.h"
RAW = re.compile(r"\b(cudaMalloc|cudaFree|cudaMallocHost|cudaFreeHost|cudaEventCreate\w*|cudaEventDestroy|cudaStreamCreate\w*|cudaStreamDestroy)\s*\(")


def test_only_the_owners_allocate_and_release():
    sources = [p for p in sorted(CSRC.iterdir()) if p.suffix in (".cu", ".cuh", ".cpp", ".h") and p != HEADER]
    assert sources
    hits = [f"{p.name}:{i}: {line.strip()}" for p in sources for i, line in enumerate(p.read_text().splitlines(), 1) if RAW.search(line)]
    assert not hits, "\n".join(hits)
    assert RAW.search(HEADER.read_text())


def test_header_compiles_on_its_own():
    gxx = shutil.which("g++")
    assert gxx, "g++ is needed to build the host code"
    cuda_inc = pathlib.Path(os.environ.get("CUDA_HOME", "/usr/local/cuda")) / "include"
    r = subprocess.run([gxx, "-std=c++17", "-fsyntax-only", "-Wall", "-Wextra", "-Werror", f"-I{cuda_inc}", f"-I{CSRC}", "-x", "c++", "-"],
                       input='#include "cuda_owned.h"\n', capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


ROUNDS_SCRIPT = textwrap.dedent("""
    import json, os, subprocess, sys
    import numpy as np
    sys.path.insert(0, sys.argv[1])
    from iris_lama_b200 import api, synth

    def used_mib():
        out = subprocess.run(["nvidia-smi", "--query-compute-apps=pid,used_memory", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, check=True).stdout
        for line in out.splitlines():
            f = [s.strip() for s in line.split(",")]
            if len(f) == 2 and f[0] == str(os.getpid()):
                return int(f[1])
        return None

    ds = synth.make_dataset("room", 3, n_beams=180)
    wall = np.array([[0.5 + 0.05 * i, 1.0, 0.3] for i in range(40)])   # inside every map's default window
    cells2, cells3 = api.w2m(0.05, wall), api.w2m3(0.05, wall)
    rng = np.random.default_rng(0)
    cloud = rng.uniform(-1.0, 1.0, (500, 3))

    def one_round():
        g = api.PFSlam2D(api.PFSlam2D.Options(4, trans_thresh=0.05, rot_thresh=0.05, seed=1))
        g.setPrior(*ds.truth[0])
        s = api.Slam2D(api.Slam2D.Options(trans_thresh=0.05, rot_thresh=0.05))
        gr = api.GraphSlam2D()
        for t in range(3):
            g.update(ds.scans[t], ds.odom[t])
            s.update(ds.scans[t], ds.odom[t])
            gr.update(ds.scans[t], ds.odom[t])
        l = api.Loc2D(api.Loc2D.Options())
        l.distance_map.addObstacle(cells2)
        l.distance_map.update()
        l.update(ds.scans[0], ds.odom[0], force_update=True)
        f = api.Loc2DFleet(api.Loc2DFleet.Options(), 2)
        f.distance_map.addObstacle(cells2)
        f.distance_map.update()
        f.update([0, 1], [ds.scans[0], ds.scans[1]], [ds.odom[0], ds.odom[1]], force=[True, True])
        dm = api.DynamicDistanceMap()
        dm.addObstacle(cells2)
        dm.update()
        om = api.FrequencyOccupancyMap()
        om.insertScans([ds.scans[0]], [[1.0, 0.0, 0.0, 0.0]])
        ts = api.TruncatedSignedDistanceMap(0.05, is3d=True)
        ts.insertPointCloud(cloud)
        o3 = api.OccupancyMap3D(0.05)
        o3.insertPointClouds([cloud])
        d3 = api.DynamicDistanceMap3D(0.05)
        d3.addObstacle(cells3)
        d3.update()
        api.pgo_optimize_graph(np.zeros((3, 3)), [(0, [0, 0, 0], api.diagonal_loss([1, 1, 1]))],
                               [(0, 1, [1, 0, 0], api.diagonal_loss([1, 1, 1])), (1, 2, [1, 0, 0], api.huber_loss(0.1))])
        try:   # refused by the shared-memory budget after every allocation of the engine was made
            api.DynamicDistanceMap(max_beams=32768)
            raise AssertionError("max_beams 32768 was not refused")
        except api.LamaError:
            pass
        del g, s, gr, l, f, dm, om, ts, o3, d3

    one_round()
    first = used_mib()
    for _ in range(99):
        one_round()
    print(json.dumps({"first": first, "last": used_mib()}))
""")


@pytest.mark.gpu
def test_handles_release_their_device_memory(gpu_api, tmp_path):
    if shutil.which("nvidia-smi") is None:
        pytest.skip("nvidia-smi is not available to read the process's device memory")
    script = tmp_path / "rounds.py"
    script.write_text(ROUNDS_SCRIPT)
    r = subprocess.run([sys.executable, str(script), str(ROOT)], capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stderr[-4000:]
    m = json.loads(r.stdout.strip().splitlines()[-1])
    if m["first"] is None or m["last"] is None:
        pytest.skip("nvidia-smi does not list this container's processes: no per-process device memory to compare")
    print(m)
    assert m["last"] - m["first"] <= 2, m   # MiB: the driver's allocation granularity
