"""Scans/s of PFSlam2D at the benchmark size with the step pipelined over G particle groups (Engine::step_groups, DESIGN.md 7a), for
G = 1 .. 4 (or the --groups given); then, in a separate profiled run per setting, the mean duration of each kernel launch, which shows how much the groups stretch each other's kernels.

  python scripts/pf_groups_rate.py [--particles 256] [--rounds 3] [--groups 1,2,3,4] [--regime revisit|forced] [--out FILE]

Timing as in bench.py's `value` (--regime revisit: scans 306 .. 405 after 300 map-building scans) or its `resample_forced` regime
(--regime forced: meas_sigma_gain 0.0008, scans 60 .. 139): staged scans, one CUDA event pair per step on the launching stream, scans/s = steps / sum of the
steps.  The settings are alternated round by round; the table gives the median and the spread over the rounds.  LAMA_PF_GROUPS is read
when an engine is created (on the first update), so each setting gets a fresh filter."""
import argparse
import json
import os
import re
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

KERNELS = ("k_match", "k_raycast", "k_brushfire")


def make_filter(api, ds, stream, P, groups, gain):
    os.environ["LAMA_PF_GROUPS"] = str(groups)
    try:
        kw = {"meas_sigma_gain": gain} if gain else {}
        pf = api.PFSlam2D(api.PFSlam2D.Options(P, trans_thresh=0.05, rot_thresh=0.05, seed=42, stream=stream.cuda_stream, **kw))
        pf.setPrior(*ds.truth[0])
        pf.stageScans(ds.scans)
        pf.updateStaged(0, ds.odom[0])   # creates the engine
    finally:
        os.environ.pop("LAMA_PF_GROUPS", None)
    return pf


def timed(torch, api, ds, stream, P, groups, first, steps, gain):
    pf = make_filter(api, ds, stream, P, groups, gain)
    for t in range(1, first):
        pf.updateStaged(t, ds.odom[t])
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(steps + 1)]
    torch.cuda.synchronize()
    ev[0].record(stream)
    for i in range(steps):
        pf.updateStaged(first + i, ds.odom[first + i])
        ev[i + 1].record(stream)
    torch.cuda.synchronize()
    ms = [ev[i].elapsed_time(ev[i + 1]) for i in range(steps)]
    st, w = pf.getParticles()
    return steps / (sum(ms) * 1e-3), float(np.median(ms)), (st.tobytes(), w.tobytes(), pf.resampleDigest())


def profiled(torch, api, ds, stream, P, groups, first, steps, gain):
    """mean device duration of each kernel over `steps` scans, from the profiler's CUDA activity records"""
    from torch.profiler import ProfilerActivity, profile
    pf = make_filter(api, ds, stream, P, groups, gain)
    for t in range(1, first):
        pf.updateStaged(t, ds.odom[t])
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(steps):
            pf.updateStaged(first + i, ds.odom[first + i])
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for k in KERNELS:
            if re.search(r"\b" + k + r"\b", e.key):
                dev = getattr(e, "device_time_total", None)
                if dev is None:
                    dev = e.cuda_time_total
                out.setdefault(k, [0.0, 0])
                out[k][0] += dev / 1000.0
                out[k][1] += e.count
    return {k: {"ms_per_scan": v[0] / steps, "launches_per_scan": v[1] / steps, "ms_per_launch": v[0] / max(v[1], 1)} for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--particles", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--prebuild", type=int, default=300)
    ap.add_argument("--profile-steps", type=int, default=30)
    ap.add_argument("--groups", default="1,2,3,4", help="comma-separated G")
    ap.add_argument("--regime", default="revisit", choices=["revisit", "forced"])
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from iris_lama_b200 import api, synth
    if api.device_count() < 1:
        raise RuntimeError("pf_groups_rate.py needs a CUDA device")
    gain = 0.0008 if a.regime == "forced" else 0.0
    first, steps = (60, 80) if a.regime == "forced" else (1 + a.prebuild + 5, a.steps)
    a.steps = steps
    ds = synth.make_dataset("loop", first + a.steps, n_beams=1080)
    stream = torch.cuda.Stream()
    settings = [int(x) for x in a.groups.split(",")]
    rates = {s: [] for s in settings}
    med = {s: [] for s in settings}
    ref = None
    for r in range(a.rounds):
        for s in (settings if r % 2 == 0 else settings[::-1]):
            v, m, res = timed(torch, api, ds, stream, a.particles, s, first, a.steps, gain)
            if ref is None:
                ref = res
            assert res[0] == ref[0] and res[1] == ref[1] and res[2] == ref[2], ("results differ from G = 1", s)
            rates[s].append(v)
            med[s].append(m)
            print(f"round {r} G={s}: {v:8.1f} scans/s  median step {m:.4f} ms", flush=True)
    prof = {}
    for s in settings:
        try:
            prof[s] = profiled(torch, api, ds, stream, a.particles, s, first, min(a.profile_steps, a.steps), gain)
        except Exception as e:   # the profiler is a diagnostic: its absence does not void the rates
            prof[s] = {"error": repr(e)}
    name = torch.cuda.get_device_name(0)
    try:
        import subprocess
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except Exception:
        pl = "unknown"
    print(f"\n{name}, power limit / max SM clock: {pl}; {a.particles} particles x 1080 beams, scans {first} .. {first + a.steps - 1} ({a.regime}), "
          f"{a.rounds} alternated rounds")
    print("G  scans/s median   min .. max        median step ms   k_match  k_raycast  k_brushfire (ms per scan, profiled)")
    base = float(np.median(rates[settings[0]]))
    rows = []
    for s in settings:
        v = np.asarray(rates[s])
        p = prof[s]
        ks = "  ".join(f"{p[k]['ms_per_scan']:.3f}" if k in p else "  -  " for k in KERNELS)
        print(f"{s}  {np.median(v):9.1f}   {v.min():7.1f} .. {v.max():7.1f}   {np.median(med[s]):.4f}"
              f"          {ks}   ({np.median(v) / base - 1:+.1%})")
        rows.append({"groups": s, "scans_per_s": v.tolist(), "median_step_ms": med[s], "kernels": p})
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump({"device": name, "power_limit_max_sm": pl, "particles": a.particles, "rows": rows, "time": time.time()}, f, indent=1)


if __name__ == "__main__":
    main()
