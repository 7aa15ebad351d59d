"""CPU restatement of lama::GraphSlam2D::update / optimizePoseGraph / getPose (src/graph_slam2d.cpp:104-430) on the test oracle's pieces:
the C++ oracle's Slam2D with a transient map and 1 m rays (pyoracle.Slam2D), its loop-closure search and scan correlation
(pyoracle.loop_closure_candidates, DDM.correlate_candidate_scan / coarse_correlate_candidate_scan) and the PGO oracle's factor graph with
Diagonal and Huber losses (pose_graph_oracle.PoseGraph).

TEST INFRASTRUCTURE ONLY: imported by tests/ and nothing else.  Besides the state of the reference class it records every decision an
update takes, with its distance to the threshold it was compared against (`margins`), so a test can tell an ill-conditioned scenario
from a real mismatch.  The function-local statics of the reference's update (odom, prev, factordist) are members, as on the device.
"""
import math

import numpy as np

from oracle import pgo_oracle as pg
from oracle import pose_graph_oracle as pgg
from oracle import pyoracle as po

DEFAULTS = dict(key_pose_distance=1.0, key_pose_angular_distance=0.5 * math.pi, key_pose_head_delay=5, loop_search_max_distance=10.0,
                loop_search_min_distance=2.0, loop_max_candidates=5, loop_closure_scan_rmse=0.05, loop_closure_max_candidates=10,
                ignore_n_chain_poses=20)   # graph_slam2d.h:62-86


def _xyr(state):
    return pg.to_xyr(np.asarray(state)[None])[0]


class GraphSlam2D:
    def __init__(self, **kw):
        self.opt = dict(DEFAULTS)
        slam_kw = {k: v for k, v in kw.items() if k not in DEFAULTS}
        self.opt.update({k: v for k, v in kw.items() if k in DEFAULTS})
        slam_kw.update(transient_map=1, truncated_ray=1.0)                 # graph_slam2d.cpp:106-107
        self.slam = po.Slam2D(po.SlamOptions.defaults(**slam_kw))
        self.keys = []          # dicts: id, pose (corrected state), original (state), pts, stamp
        self.links = []
        self.priors, self.factors, self.queue = [], [], []
        self.correction = pg.from_xyr([0.0, 0.0, 0.0])[0]
        self.accdist = 0.0
        self.prev = pg.from_xyr([1e10, 1e10, 0.0])[0]
        self.factordist = 0.0
        self.decisions = []     # one record per update that reached the key-pose test
        self.margins = []       # (what, |value - threshold|)
        self.optimizations = []

    def Init(self, x, y, r):
        self.slam.set_pose(x, y, r)

    def getPose(self):
        return _xyr(pg.mul(self.correction[None], self.slam.state()[None])[0])

    def update(self, pts, odom, stamp=0.0):
        if not self.slam.update(pts, odom):
            return False
        o = self.opt
        sp = self.slam.state()
        diff = pg.mul(pg.inv(sp[None]), self.prev[None])[0]                 # slam pose - prev (pose2d.cpp:81-84)
        dxy, drot = math.hypot(diff[2], diff[3]), math.atan2(diff[1], diff[0])
        self.margins.append(("key_distance", abs(dxy - o["key_pose_distance"])))
        if dxy < o["key_pose_distance"]:   # the angle is compared only then (&&, graph_slam2d.cpp:203-204)
            self.margins.append(("key_angle", abs(abs(drot) - o["key_pose_angular_distance"])))
        rec = dict(stamp=stamp, key=None, searched=False, candidates=[], correlations=[], link=None, queue=0, factordist=0.0, flush=False, pgo=None)
        self.decisions.append(rec)
        if dxy < o["key_pose_distance"] and abs(drot) < o["key_pose_angular_distance"]:
            return True
        self.prev = sp
        keyid = len(self.keys)
        corrected = pg.mul(self.correction[None], sp[None])[0]
        if keyid == 0:
            self.priors.append((0, _xyr(sp), pgg.diagonal([0.01, 0.01, 0.01])))
        else:
            self.accdist += dxy
            between = pg.mul(pg.inv(self.keys[-1]["pose"][None]), corrected[None])[0]
            self.factors.append((keyid - 1, keyid, _xyr(between), pgg.diagonal([0.25, 0.25, 0.15])))
        self.keys.append(dict(id=keyid, pose=corrected, original=sp, pts=np.array(pts, float), stamp=stamp))
        rec["key"] = keyid
        if keyid < o["key_pose_head_delay"] or keyid < o["ignore_n_chain_poses"]:
            return True

        r = min(self.accdist, 100.0) / 100.0
        radius = o["loop_search_max_distance"] ** r * o["loop_search_min_distance"] ** (1.0 - r)
        keyid -= o["key_pose_head_delay"]
        key_xy = np.array([k["pose"][2:4] for k in self.keys])
        query = self.keys[keyid]["pose"][2:4]
        cands = [int(c) for c in po.loop_closure_candidates(key_xy, o["ignore_n_chain_poses"], query, radius, o["loop_max_candidates"])]
        rec["searched"], rec["candidates"] = True, cands
        d = np.sqrt(((key_xy[:len(self.keys) - o["ignore_n_chain_poses"]] - query) ** 2).sum(1))
        if len(d):
            self.margins.append(("search_radius", float(np.abs(d - radius).min())))
            ds = np.sort(d[d < radius])
            if len(ds) > o["loop_max_candidates"]:
                self.margins.append(("candidate_cap", float(ds[o["loop_max_candidates"]] - ds[o["loop_max_candidates"] - 1])))
        self.factordist += dxy

        cinv = pg.inv(self.correction[None])
        ref = self.keys[keyid]
        ref_xyr = _xyr(pg.mul(cinv, ref["pose"][None])[0])
        dm = self.slam.dm()
        thr = o["loop_closure_scan_rmse"]
        for i, idx in enumerate(cands):
            cand = self.keys[idx]
            cand_xyr = _xyr(pg.mul(cinv, cand["pose"][None])[0])
            between, rmse = dm.correlate_candidate_scan(cand["pts"], ref_xyr, cand_xyr)
            self.margins.append(("scan_rmse", abs(rmse - thr)))
            corr = dict(candidate=idx, rmse=rmse, coarse_rmse=None)
            rec["correlations"].append(corr)
            if rmse > thr:
                if i != 0:
                    continue
                between, rmse = dm.coarse_correlate_candidate_scan(ref["pts"], cand["pts"], ref_xyr, cand_xyr)   # :254-258
                corr["coarse_rmse"] = rmse
                self.margins.append(("coarse_scan_rmse", abs(rmse - 2.0 * thr)))
                if rmse > thr * 2.0:
                    continue
            self.links.append((idx, keyid))
            self.queue.append((idx, keyid, np.array(between), pgg.huber(0.1)))   # HuberLoss::Huber(0.1), :266-268
            rec["link"] = (idx, keyid)
            self.factordist = 0.0
            break
        rec["queue"], rec["factordist"] = len(self.queue), self.factordist
        if self.queue and len(self.queue) <= 5:
            self.margins.append(("flush_distance", abs(self.factordist - 15.0)))
        if not self.queue or (len(self.queue) <= 5 and self.factordist <= 15.0):
            return True
        rec["flush"] = True
        rec["pgo"] = self.optimizePoseGraph()
        self.factordist = 0.0
        return True

    def optimizePoseGraph(self):
        """:394-430 -> (status, iterations, lambda_tries, accepted flags)"""
        if not self.queue:
            return None
        self.factors += self.queue
        self.queue = []
        g = pgg.PoseGraph(np.array([_xyr(k["pose"]) for k in self.keys]), self.priors, self.factors)
        g.optimize()
        if g.status == 0:
            for i, k in enumerate(self.keys):
                k["pose"] = g.nodes[i].copy()
            A, B = self.keys[-1]["pose"], self.slam.state()
            self.correction = pg.inv(pg.mul(B[None], pg.inv(A[None])))[0]
        self.accdist = 0.0
        out = (g.status, g.iterations, g.lambda_tries, list(g.accepted))
        self.optimizations.append(out)
        return out

    def key_poses(self):
        """(corrected n x 3, original n x 3) as xyr"""
        return (np.array([_xyr(k["pose"]) for k in self.keys]).reshape(-1, 3), np.array([_xyr(k["original"]) for k in self.keys]).reshape(-1, 3))
