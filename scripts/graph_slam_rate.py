"""GraphSlam2D on the device over the two-lap loop world (synth "loop", 1600 scans, 1080 beams): updates per second of the whole run
(host clock around GraphSlam2D.update, each update ends in a device synchronise), and the device time and CG iterations of every pose-graph
optimisation it ran.  Prints one JSON line with the card's name and power limit; writes it to OUT_DIR/graph_slam_rate.json when given."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from iris_lama_b200 import api, synth  # noqa: E402


def main():
    out_dir = sys.argv[1] if len(sys.argv) > 1 else None
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    ds = synth.make_dataset("loop", 1600, n_beams=1080)
    runs = []
    for rep in range(2):   # the first run also pays module loading and allocation; the second is the figure
        g = api.GraphSlam2D()
        g.Init(*ds.truth[0])
        opts, n_upd = [], 0
        t0 = time.perf_counter()
        for t in range(ds.n_scans):
            did = g.update(ds.scans[t], ds.odom[t], float(t))
            n_upd += int(did)
            st = g.stats()
            if st["optimizations"] > len(opts):
                opts.append(dict(status=st["last_status"], keys=st["key_poses"], **{k: st["last_report"][k] for k in ("iterations", "cg_iterations", "device_ms")}))
        dt = time.perf_counter() - t0
        st = g.stats()
        runs.append(dict(scans=ds.n_scans, updates=n_upd, seconds=dt, scans_per_s=ds.n_scans / dt, updates_per_s=n_upd / dt, key_poses=st["key_poses"],
                         loop_factors=st["loop_factors"], optimizations=opts))
    res = dict(card=card, first_run=runs[0], run=runs[1])
    line = json.dumps(res)
    print(line)
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "graph_slam_rate.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
