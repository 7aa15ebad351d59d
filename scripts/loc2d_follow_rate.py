"""Rates of Loc2D on a following distance map (lama_dm_set_follow) on the device.

- Tracking: Loc2D (cov_blend 0.5, updates every 0.2 m) out and back along an 84 m corridor, the map read from the oracle's file, on a
  following dir_dim 16 map (25.6 m windows, patches parked) and on a fixed dir_dim 128 map that holds it all: updates per second, wall
  clock over the whole path (every update ends in a synchronisation), median of REPEATS runs on fresh handles.
- Global localisation: device time of one 3000-candidate scoring launch, from CUDA events around the match launches (dev timing): the
  match time of an update with a global-localisation step minus that of the following tracking-only update.  On a following dir_dim 128
  map of a 300 m corridor (k_match_extent over the whole map) and on the 84 m corridor in a fixed dir_dim 128 window (k_match).
- The wall time of reading the 300 m map into the following map (lama_dm_read: parse, tiles, window shifts).
- The oracle's single-thread time for the same global-localisation step (host clock: oracle update with the step minus without).

Prints one JSON line with the card's name and power limit; writes it to OUT_DIR/loc2d_follow_rate.json when given."""
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from iris_lama_b200 import api, synth  # noqa: E402
from oracle import pyoracle as po  # noqa: E402
from test_gpu_window_follow import _out_and_back  # noqa: E402
from test_gpu_loc2d_follow import _cells, _free  # noqa: E402

REPEATS = 3
KW = dict(trans_thresh=0.2, rot_thresh=0.2, cov_blend=0.5)


def oracle_file(cells, path):
    od = po.DDM(0.05, 32, 1.0)
    od.add(cells)
    od.update()
    assert po.map_write("ddm", od, path)


def loc(path, dir_dim, follow, **kw):
    g = api.Loc2D(api.Loc2D.Options(dir_dim=dir_dim, max_beams=512, **KW, **kw))
    if follow:
        g.distance_map.setFollow(True)
    t = time.perf_counter()
    g.distance_map.read(path)
    return g, time.perf_counter() - t


def tracking_rate(path, truth, odom, scans, dir_dim, follow):
    rates, windows = [], None
    for _ in range(REPEATS):
        g, _ = loc(path, dir_dim, follow)
        g.setPose(*truth[0])
        g.update(scans[0], odom[0], force_update=True)
        t = time.perf_counter()
        n = sum(g.update(scans[k], odom[k]) for k in range(1, len(scans)))
        rates.append(n / (time.perf_counter() - t))
        windows = g.distance_map.window()
    return statistics.median(rates), windows


def gloc_times(path, length, truth, odom, scans, t0, dir_dim, follow):
    """device ms of the 3000-candidate launch per step, and (oracle) host ms of the step"""
    cells_free = _free(length)
    dev, orc = [], []
    for rep in range(REPEATS):
        g, _ = loc(path, dir_dim, follow, gloc_particles=3000, timing=1)
        g.occupancySet(cells_free, -1); g.setSeed(rep + 1)
        x, y, r = truth[t0]
        g.setPose(x, y, r)
        g.update(scans[t0], odom[t0], force_update=True)
        g.triggerGlobalLocalization()
        with_step = None
        for k in range(t0 + 1, t0 + 14):   # the last step with global localisation, then the first without (at most gloc_iters steps)
            m0 = g.distance_map.kernelTimes()[0]["match_ms"]
            active = g.globalLocalizationActive()
            g.update(scans[k], odom[k], force_update=True)
            ms = g.distance_map.kernelTimes()[0]["match_ms"] - m0
            if active:
                with_step = ms
            elif with_step is not None:
                dev.append(with_step - ms)
                break
    for rep in range(REPEATS):
        ol = po.Loc2D(po.LocOptions.defaults(gloc_particles=3000, **KW))
        ol.occ_set(cells_free, -1)
        assert po.map_read("ddm", ol.dm(), path)
        ol.set_seed(rep + 1)
        ol.set_pose(*truth[t0])
        ol.update(scans[t0], odom[t0], force=True)
        t = time.perf_counter()
        ol.update(scans[t0 + 1], odom[t0 + 1], force=True)
        plain = time.perf_counter() - t
        ol.trigger_global_localization()
        t = time.perf_counter()
        ol.update(scans[t0 + 1], odom[t0 + 1], force=True)
        orc.append((time.perf_counter() - t - plain) * 1e3)
    return (statistics.median(dev) if dev else None), statistics.median(orc)


def main():
    if api.device_count() < 1:
        raise SystemExit("needs a CUDA device")
    tmp = tempfile.mkdtemp()
    out = {}
    truth, odom, scans = _out_and_back(synth)
    short = os.path.join(tmp, "corridor84.sdm")
    oracle_file(_cells(synth.make_corridor(length=84.0)), short)
    for name, dim, follow in (("following_dir16", 16, True), ("fixed_dir128", 128, False)):
        rate, w = tracking_rate(short, truth, odom, scans, dim, follow)
        out[f"tracking_updates_per_s_{name}"] = round(rate, 1)
        out[f"tracking_window_{name}"] = w
    ltruth, lodom, lscans = _out_and_back(synth, length=300.0, step=0.5)
    long_ = os.path.join(tmp, "corridor300.sdm")
    oracle_file(_cells(synth.make_corridor(length=300.0)), long_)
    reads = []
    for _ in range(REPEATS):
        g, s = loc(long_, 128, True)
        reads.append(s * 1e3)
    out["read_300m_ms"] = round(statistics.median(reads), 2)
    out["read_300m_window"] = g.distance_map.window()
    out["read_300m_pool"] = g.distance_map.pool()
    t0 = len(ltruth) // 2 - 40
    dev, orc = gloc_times(long_, 300.0, ltruth, lodom, lscans, t0, 128, True)
    out["gloc_3000_device_ms_300m_following_dir128"] = None if dev is None else round(dev, 3)
    out["gloc_3000_oracle_ms_300m"] = round(orc, 1)
    dev, orc = gloc_times(short, 84.0, truth, odom, scans, 100, 128, False)
    out["gloc_3000_device_ms_84m_fixed_dir128"] = None if dev is None else round(dev, 3)
    out["gloc_3000_oracle_ms_84m"] = round(orc, 1)
    out["card"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                                 text=True).stdout.strip()
    line = json.dumps(out)
    print(line)
    out_dir = os.environ.get("OUT_DIR")
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "loc2d_follow_rate.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
