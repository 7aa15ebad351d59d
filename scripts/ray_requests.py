"""Host model of the counter reductions of k_raycast's walk: for every RED instruction of one particle's ray cast, the distinct cells,
32-byte sectors and 128-byte lines it touches, in the issue order of raycast_pass without (`current`) and with (`aligned`) the sector-aligned
segments of x-major beams in x-major groups.  CPU only; no time is measured or implied.

The beams are the bench's (`synth.make_dataset("loop", ...)`, 1080 beams) cast from the TRUE pose, not from the particles' poses, and
world -> map uses floor(x * 20 + 0.5), so the cells differ slightly from the device's; only the order of the walk is modelled exactly.

  python scripts/ray_requests.py [scan ...]        (default: scans 306 355 405, the first, middle and last timed scans of bench.py)
"""
import math
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from iris_lama_b200 import synth  # noqa: E402

SEG, STRIDE, SCALE = 64, 8, 20.0


def beams_of(ds, t):
    x, y, th = ds.truth[t]
    p = ds.scans[t]
    hx = x + math.cos(th) * p[:, 0] - math.sin(th) * p[:, 1]
    hy = y + math.sin(th) * p[:, 0] + math.cos(th) * p[:, 1]
    w2m = lambda v: np.floor(v * SCALE + 0.5).astype(np.int64)  # noqa: E731
    fx, fy = int(w2m(np.array([x]))[0]), int(w2m(np.array([y]))[0])
    return np.full(len(p), fx), np.full(len(p), fy), w2m(hx), w2m(hy)


class Beams:
    def __init__(self, fx, fy, tx, ty):
        self.fx, self.fy, self.tx, self.ty = fx, fy, tx, ty
        dx, dy = tx - fx, ty - fy
        self.xmajor = np.abs(dx) >= np.abs(dy)
        self.n = np.maximum(np.abs(dx), np.abs(dy))
        self.d = np.minimum(np.abs(dx), np.abs(dy))
        self.sx, self.sy = np.where(dx < 0, -1, 1), np.where(dy < 0, -1, 1)
        self.shift = np.where(dx < 0, -fx, fx + 1) & 7   # ray_core.h xmajor_seg_shift

    def cells(self, b, i):   # closed form of the planar Bresenham state after i steps (ray_core.h SegWalk)
        n, d = self.n[b], self.d[b]
        k = (2 * i * d + n) // np.maximum(2 * n, 1)
        maj, mnr = self.sx[b] * i, np.where(self.xmajor[b], self.sy[b], self.sx[b]) * k
        return (np.where(self.xmajor[b], self.fx[b] + maj, self.fx[b] + mnr),
                np.where(self.xmajor[b], self.fy[b] + mnr, self.fy[b] + self.sy[b] * i))


def address(x, y):   # byte address with every patch of 32 x 32 counters at its own 4 KiB
    return (((y >> 5) * 65536 + (x >> 5)) << 12) | ((x & 31) << 2) | ((y & 31) << 7)


def requests(B, aligned):
    """(class, instruction id, beam, step) of every RED lane; classes: 0 hits, 1 segment 0, 2 y-major groups, 3 x-major groups"""
    out = []
    iid = 0
    N = len(B.n)

    def emit(cls, ids, beam, step, ok):
        out.append((np.full(ok.sum(), cls), ids[ok], beam[ok], step[ok]))

    for g0 in range(0, N, 32):
        bs = np.arange(g0, min(g0 + 32, N))
        emit(0, np.full(len(bs), iid), bs, np.zeros(len(bs), np.int64), np.ones(len(bs), bool))
        iid += 1
    for g0 in range(0, N, 32):
        bs = np.arange(g0, min(g0 + 32, N))
        xg = 2 * B.xmajor[bs].sum() > len(bs)
        delta = np.where(B.xmajor[bs], B.shift[bs], 0) if aligned and xg else np.zeros(len(bs), np.int64)
        walk = B.n[bs] - 1
        segs = int(np.max(np.where(walk > 0, (walk + delta + SEG - 1) // SEG, 0)))
        if segs == 0:
            continue
        # segment 0: lane = beam, steps 1 .. 64 - delta in lock step; runs of equal cells in adjacent lanes issue one RED
        t = np.arange(1, SEG + 1)[:, None]
        lanes = np.broadcast_to(bs, (SEG, len(bs)))
        steps = np.broadcast_to(t, lanes.shape)
        ok = steps <= np.minimum(SEG - delta, walk)
        x, y = B.cells(lanes, steps)
        key = np.where(ok, x * 1000003 + y, -1)
        head = ok & np.concatenate([np.ones((SEG, 1), bool), (key[:, 1:] != key[:, :-1]) | ~ok[:, :-1]], axis=1)
        emit(1, (iid + t - 1 + 0 * lanes).ravel(), lanes.ravel(), steps.ravel(), head.ravel())
        iid += SEG
        for s in range(1, segs):
            if not xg:   # lane = beam, one step at a time
                steps = s * SEG + t + 0 * lanes
                emit(2, (iid + t - 1 + 0 * lanes).ravel(), lanes.ravel(), steps.ravel(), (steps <= walk).ravel())
                iid += SEG
                continue
            for r in range(STRIDE):   # 4 beams x 8 lanes at consecutive offsets, stride 8
                q = np.arange(r * (32 // STRIDE), (r + 1) * (32 // STRIDE))
                q = q[q < len(bs)]
                if len(q) == 0:
                    continue
                first = s * SEG + 1 - delta[q]
                j = np.arange(SEG // STRIDE)[:, None, None]
                k = np.arange(STRIDE)[None, None, :]
                steps = first[None, :, None] + k + STRIDE * j
                ok = steps <= np.minimum(first + SEG - 1, walk[q])[None, :, None]
                beam = np.broadcast_to(bs[q][None, :, None], steps.shape)
                emit(3, np.broadcast_to(iid + j, steps.shape).ravel(), beam.ravel(), steps.ravel(), ok.ravel())
                iid += SEG // STRIDE
    cls, ids, beam, step = (np.concatenate(v) for v in zip(*out))
    hx, hy = B.tx[beam], B.ty[beam]
    x, y = B.cells(beam, step)
    x, y = np.where(step == 0, hx, x), np.where(step == 0, hy, y)
    return cls, ids, address(x, y)


def distinct(ids, key):
    return len(np.unique(np.stack([ids, key]), axis=1)[0])


def main():
    scans = [int(a) for a in sys.argv[1:]] or [306, 355, 405]
    ds = synth.make_dataset("loop", max(scans) + 1, n_beams=1080)
    names = ["hits", "segment 0", "y-major groups, segments >= 1", "x-major groups, segments >= 1"]
    print("per particle per scan: RED lanes / distinct cells / sectors / lines summed over instructions")
    for t in scans:
        B = Beams(*beams_of(ds, t))
        res = {}
        for order in ("current", "aligned"):
            cls, ids, addr = requests(B, order == "aligned")
            rows = []
            for c in range(4):
                m = cls == c
                rows.append((m.sum(), distinct(ids[m], addr[m]), distinct(ids[m], addr[m] >> 5), distinct(ids[m], addr[m] >> 7)))
            res[order] = rows
        print(f"scan {t}:")
        for c, name in enumerate(names):
            a, b = res["current"][c], res["aligned"][c]
            print(f"  {name:32s} current {a[0]:7d} / {a[1]:7d} / {a[2]:7d} / {a[3]:7d}   aligned {b[0]:7d} / {b[1]:7d} / {b[2]:7d} / {b[3]:7d}")
        sa, sb = sum(r[2] for r in res["current"]), sum(r[2] for r in res["aligned"])
        print(f"  all sectors: current {sa}, aligned {sb} ({100.0 * (sb - sa) / sa:+.1f} %)")


if __name__ == "__main__":
    main()
