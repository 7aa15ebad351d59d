"""Checkpoint cost on the bench workload: PFSlam2D 256 particles x 1080 beams on the synthetic loop, forced resampling (meas_sigma_gain
0.0008), saved after scan `--scans`, loaded back, then both handles continue `--continue` scans and must report the same.

Prints one JSON line: the card's name and power limit (read in the same run), used slots against the per-particle patch references
(the dedupe factor of the copy-on-write sharing), file bytes, the snapshot split into count / compaction / gather (CUDA events) and
copy-out (host clock of the chunked copy through pinned buffers), the restore split into engine creation / tables / copy-in, host I/O
apart, and gather / copy throughput against the HBM3 data-sheet figure and the measured host link.  With --out, the same result also goes
to DIR/checkpoint_rate.json.

    python scripts/checkpoint_rate.py [--scans 400] [--continue 20] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_TBS = 3.35   # NVIDIA H100 SXM data sheet, HBM3


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], text=True)
        name, power, clock = [v.strip() for v in out.splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:   # the numbers below are still device times; the card stays unnamed
        return {"name": None, "error": str(e)}


def host_link_gbs():
    """pinned host <-> device copy rate of the host and card in use (torch, 256 MiB)"""
    import torch
    n = 256 << 20
    d = torch.empty(n, dtype=torch.uint8, device="cuda")
    h = torch.empty(n, dtype=torch.uint8, pin_memory=True)
    out = {}
    for name, (dst, src) in {"d2h": (h, d), "h2d": (d, h)}.items():
        dst.copy_(src, non_blocking=True)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(5):
            dst.copy_(src, non_blocking=True)
        torch.cuda.synchronize()
        out[name] = 5 * n / (time.perf_counter() - t0) / 1e9
    return out


def state(g, particles):
    st, w = g.getParticles()
    d = dict(states=st.tobytes(), weights=w.tobytes(), neff=g.getNeff(), best=g.getBestParticleIdx(), last=g.lastResample().tolist(),
             digest=g.resampleDigest(), mem=g.getMemoryUsage())
    # the work counters without `detached`, which counts copy-on-write races and differs between any two runs (DESIGN.md §13)
    d["counters"] = tuple({k: v for k, v in c.items() if k != "detached"} for c in g.counters())
    for p in particles:
        for kind in (0, 1):
            n, mn, mx = g.mapBounds(p, kind)
            d[(p, kind)] = (n, mn.tolist(), mx.tolist())
            if n:
                w_, h_ = int(mx[0] - mn[0]), int(mx[1] - mn[1])
                e = g.exportOccupancy(p, mn[0], mn[1], w_, h_) if kind == 0 else g.exportDistance(p, mn[0], mn[1], w_, h_)
                d[(p, kind, "cells")] = {k: v.tobytes() for k, v in e.items()}
    return d


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=400)
    ap.add_argument("--continue", dest="cont", type=int, default=20)
    ap.add_argument("--particles", type=int, default=256)
    ap.add_argument("--out", default=None, help="directory for checkpoint_rate.json (default: print only)")
    a = ap.parse_args()
    from iris_lama_b200 import api, synth
    if api.device_count() < 1:
        raise SystemExit("checkpoint_rate.py needs a CUDA device: the lama_b200 hot path has no CPU fallback")
    ds = synth.make_dataset("loop", a.scans + a.cont, n_beams=1080)
    g = api.PFSlam2D(api.PFSlam2D.Options(a.particles, trans_thresh=0.05, rot_thresh=0.05, seed=42, meas_sigma_gain=0.0008))
    g.setPrior(*ds.truth[0])
    for t in range(a.scans):
        g.update(ds.scans[t], ds.odom[t])
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "pf.ckpt")
        saves, loads = [], []
        for rep in range(3):   # the first round warms the allocator and the page cache; the reported numbers are the last round's
            g.saveState(path)
            saves.append(api.checkpoint_stats())
            b = api.PFSlam2D.loadState(path)
            loads.append(api.checkpoint_stats())
            assert b.counters() == g.counters()
            if rep < 2:
                del b
        s, l = saves[-1], loads[-1]
        for t in range(a.scans, a.scans + a.cont):
            assert g.update(ds.scans[t], ds.odom[t]) == b.update(ds.scans[t], ds.odom[t])
            assert state(g, (0, 101, a.particles - 1)) == state(b, (0, 101, a.particles - 1)), t
        for i in range(a.particles):
            assert (g.trajectory(i) == b.trajectory(i)).all()
    link = host_link_gbs()
    slot_bytes = s["used_slots"] * (4096 + 128)
    res = {
        "workload": f"PFSlam2D {a.particles} x 1080, loop, meas_sigma_gain 0.0008, saved after {a.scans} scans, {a.cont} scans continued: equal",
        "card": card(), "resamplings": g.resampleDigest()[0],
        "used_slots": s["used_slots"], "patch_references": s["references"], "dedupe": s["references"] / max(1, s["used_slots"]),
        "file_bytes": s["file_bytes"],
        "snapshot_ms": {k: s[k] for k in ("count_ms", "compact_ms", "gather_ms", "copy_ms")},
        "save_host_ms": {"encode": s["encode_ms"], "write": s["io_ms"], "total": s["total_ms"]},
        "restore_ms": {k: l[k] for k in ("create_ms", "tables_ms", "copy_ms")},
        "load_host_ms": {"read": l["io_ms"], "decode_and_check": l["encode_ms"], "total": l["total_ms"]},
        "gather_TBps": 2 * slot_bytes / (s["gather_ms"] * 1e-3) / 1e12 if s["gather_ms"] > 0 else None,   # read + write of the slot bytes
        "gather_of_hbm_peak": (2 * slot_bytes / (s["gather_ms"] * 1e-3) / 1e12) / HBM_TBS if s["gather_ms"] > 0 else None,
        "copy_out_GBps": slot_bytes / (s["copy_ms"] * 1e-3) / 1e9 if s["copy_ms"] > 0 else None,
        "copy_in_GBps": slot_bytes / (l["copy_ms"] * 1e-3) / 1e9 if l["copy_ms"] > 0 else None,
        "host_link_GBps": link, "all_rounds": {"save": saves, "load": loads},
    }
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "checkpoint_rate.json"), "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
