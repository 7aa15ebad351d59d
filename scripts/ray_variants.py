"""Developer experiment (LAMA_PHASE_TIMING build): k_raycast time with reductions / the LDS removed, after 300 correct scans.
LAMA_RAY_DEBUG: 0 everything, 1 no RED, 2 no LDS (3 neither), 4 no RED in x-major beam groups, 8 no RED in y-major beam groups.
The build prints one line per launch for CTAs 0 and 200 (phase cycles, walk cells per group class, tagged with the debug value);
this script prints the ray-cast time per scan of each window and, at the end, the median phase cycles of each debug value."""
import collections, os, re, statistics, subprocess, sys, tempfile
sys.path.insert(0, '.')

if os.environ.get("_RAY_VARIANTS_CHILD") != "1":   # run the experiment in a child so the device printf lines can be collected
    with tempfile.TemporaryFile("w+") as out:
        rc = subprocess.call([sys.executable, __file__] + sys.argv[1:], stdout=out, stderr=subprocess.STDOUT,
                             env=dict(os.environ, _RAY_VARIANTS_CHILD="1"))
        out.seek(0)
        phases = collections.defaultdict(list)
        for line in out:
            m = re.match(r"ray cta \d+ debug (\d+): setup (\d+) walk (\d+) sort (\d+) replay (\d+) events (\d+) .*y-major (\d+) x-major (\d+)", line)
            if m:
                phases[int(m.group(1))].append([int(v) for v in m.groups()[1:]])
            elif not line.startswith("ray cta"):
                print(line, end="")
    for dbg, rows in sorted(phases.items()):
        rows = rows[-40:]   # the last window run with this value (revisit scans)
        med = [statistics.median(col) for col in zip(*rows)]
        print("debug %d phase cycles (median of %d CTA launches): setup %d walk %d sort %d replay %d events %d | walk cells y-major %d x-major %d"
              % (dbg, len(rows), *med))
    sys.exit(rc)

from iris_lama_b200 import api, synth
ds = synth.make_dataset("loop", 400, n_beams=1080)
g = api.PFSlam2D(api.PFSlam2D.Options(256, trans_thresh=0.05, rot_thresh=0.05, seed=42, timing=1))
g.setPrior(*ds.truth[0])
def run(t0, t1):
    g.getPose(); a, _ = g.kernelTimes()
    for t in range(t0, t1): g.update(ds.scans[t], ds.odom[t])
    g.getPose(); b, _ = g.kernelTimes()
    return {k: (b[k] - a[k]) / (t1 - t0) for k in a}
run(0, 300)
t = 300
for dbg in (0, 1, 4, 8, 0):
    os.environ["LAMA_RAY_DEBUG"] = str(dbg)
    print("debug", dbg, "scans", t, t + 20, run(t, t + 20), flush=True)
    t += 20
