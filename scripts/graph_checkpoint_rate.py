"""Checkpoint cost of a GraphSlam2D session: two laps of the synthetic 30 m loop room (1 600 scans, 1 080 beams), a full-resolution global
map generated at the end, then saved and loaded three times; the loaded handle and the saved one continue `--continue` scans and must
report the same.

Prints one JSON line: the card's name and power limit (read in the same run), the session's counts at the save, the checkpoint_stats()
split of the last save and load round (device times and slots are sums over the inner Slam2D's engine and the global map's engine), and
the file's bytes per section with the slots of each engine, read back from the saved file; the sections must add up to its size.  With --out, the same result also goes to DIR/graph_checkpoint_rate.json.

    python scripts/graph_checkpoint_rate.py [--continue 40] [--out DIR]
"""
import argparse
import json
import os
import struct
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N_SCANS, BEAMS = 1600, 1080


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], text=True)
        name, power, clock = [v.strip() for v in out.splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:   # the numbers below are still device times; the card stays unnamed
        return {"name": None, "error": str(e)}


def file_sections(data):
    """bytes per section of a kind-4 file, read from the file itself (DESIGN.md §13), and the slots, known plane and directory size of
    each engine; the sections must add up to the file"""
    off = 32
    out = {"header": 32}

    def take(name, n):
        nonlocal off
        out[name] = out.get(name, 0) + n
        off += n
        return data[off - n:off]

    def u32(name):
        return struct.unpack("<I", take(name, 4))[0]

    take("graph_options", 56)
    take("inner_slam_options_and_state", 292)
    take("graph_state", 4 * 8 * 2 + 2 * 8 + 8 + 3 * 8 + 44)
    take("graph_state", 4 * u32("graph_state") + 16)
    for _ in range(u32("key_poses")):
        take("key_poses", 136)
        take("key_clouds", 24 * struct.unpack("<I", data[off - 4:off])[0])
    take("links", 8 * u32("links"))
    take("pose_graph", 68 * u32("pose_graph"))
    take("pose_graph", 72 * u32("pose_graph"))
    take("pose_graph", 72 * u32("pose_graph"))
    engines = {}
    for name in ("inner_engine", "global_map"):
        if take(name, 1) == b"\x00":
            continue
        particles, dir_dim, _, _, kind = struct.unpack("<5i", take(name, 20))
        known = take(name, 1) == b"\x01"
        take(name, 16 + 8 + 24)
        K = u32(name)
        n_dir = particles * (3 if kind == 1 else 2) * dir_dim * dir_dim
        take(name, 4 * K + 4 * n_dir)
        take(name + "_slots", K * (4096 + 128 + (128 if known or kind == 1 else 0)))
        engines[name] = {"slots": K, "dir_dim": dir_dim, "known_plane": known}
    if off != len(data):
        raise SystemExit(f"the sections of the saved file add up to {off} bytes, the file has {len(data)}")
    return out, engines


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--continue", dest="cont", type=int, default=40)
    ap.add_argument("--out", default=None, help="directory for graph_checkpoint_rate.json (default: print only)")
    a = ap.parse_args()
    from iris_lama_b200 import api, synth
    if api.device_count() < 1:
        raise SystemExit("graph_checkpoint_rate.py needs a CUDA device: the lama_b200 hot path has no CPU fallback")

    def check(ok, what):   # not an assert: the result line claims these, so they are checked under python -O too
        if not ok:
            raise SystemExit(f"graph_checkpoint_rate.py: {what}")

    ds = synth.make_dataset("loop", N_SCANS + a.cont, n_beams=BEAMS)
    g = api.GraphSlam2D()
    g.Init(*ds.truth[0])
    for t in range(N_SCANS):
        g.update(ds.scans[t], ds.odom[t], float(t))
    g.generateOccupancyMap(full=True)
    st = g.stats()   # the saved state: everything below describes the session at the save, not after the continuation
    n_keys = st["key_poses"]
    cloud_bytes = sum(g.keyCloud(i)[0].nbytes for i in range(n_keys))
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "graph.ckpt")
        saves, loads = [], []
        for rep in range(3):   # the first round warms the allocator and the page cache; the reported numbers are the last round's
            g.saveState(path)
            saves.append(api.checkpoint_stats())
            b = api.GraphSlam2D.loadState(path)
            loads.append(api.checkpoint_stats())
            check(b.stats() == g.stats(), f"round {rep}: the loaded handle's stats differ from the saved one's")
            if rep < 2:
                del b
        s, l = saves[-1], loads[-1]
        with open(path, "rb") as f:
            data = f.read()
        check(len(data) == s["file_bytes"], "checkpoint_stats() file_bytes differs from the file's size")
        sections, engines = file_sections(data)
        check(sections.get("key_clouds", 0) == cloud_bytes, "the key clouds in the file differ from keyCloud()")
        check(sum(e["slots"] for e in engines.values()) == s["used_slots"], "the slots in the file differ from checkpoint_stats()")
        for t in range(N_SCANS, N_SCANS + a.cont):
            check(g.update(ds.scans[t], ds.odom[t], float(t)) == b.update(ds.scans[t], ds.odom[t], float(t)), f"update {t} differs")
            check((g.getPose() == b.getPose()).all(), f"pose after update {t} differs")
        # device_ms of an optimisation run after the load is a timing, not state: it differs between any two runs
        strip = lambda d: dict(d, last_report={k: v for k, v in d["last_report"].items() if k != "device_ms"})
        check((g.keyPoses()[0] == b.keyPoses()[0]).all() and strip(g.stats()) == strip(b.stats()), "key poses or stats differ after the continuation")
    res = {
        "workload": f"GraphSlam2D, loop, {N_SCANS} scans x {BEAMS} beams, generateOccupancyMap(full=True) at the end; saved, loaded, "
                    f"{a.cont} scans continued: equal",
        "card": card(),
        "at_save": {"key_poses": n_keys, "loop_factors": st["loop_factors"], "optimizations": st["optimizations"]},
        "file_bytes": s["file_bytes"], "key_cloud_bytes": cloud_bytes, "section_bytes": sections, "engines": engines,
        "slots": s["used_slots"], "references": s["references"],
        "snapshot_ms": {k: s[k] for k in ("count_ms", "compact_ms", "gather_ms", "copy_ms")},
        "save_host_ms": {"encode": s["encode_ms"], "write": s["io_ms"], "total": s["total_ms"]},
        "restore_ms": {k: l[k] for k in ("create_ms", "tables_ms", "copy_ms")},
        "load_host_ms": {"read": l["io_ms"], "decode_and_check": l["encode_ms"], "total": l["total_ms"]},
        "all_rounds": {"save": saves, "load": loads},
    }
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "graph_checkpoint_rate.json"), "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
