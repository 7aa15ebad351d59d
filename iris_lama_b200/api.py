"""Python host mirror of the reference front ends over the C-ABI (include/lama_b200.h).

Class and method names follow the reference (lama::PFSlam2D / Slam2D / Loc2D / DynamicDistanceMap,
include/lama/*.h) so parity tests read like tests of the reference.  Every call goes through
liblama_b200.so; there is no CPU fallback: without the CUDA extension or without a GPU the
constructors raise.
"""
from __future__ import annotations

import ctypes as C
import os
import struct

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("LAMA_B200_LIB") or os.path.join(_HERE, "liblama_b200.so")   # the override is for developer builds of the same library
_lib = None

c_dp = C.POINTER(C.c_double)
c_u32p = C.POINTER(C.c_uint32)
c_i32p = C.POINTER(C.c_int32)
c_u64p = C.POINTER(C.c_uint64)

OFFSET = 1321122 * 32  # map-cell coordinate of world 0.0 (include/lama/sdm/map.h:68, src/sdm/map.cpp:55-58)


class LamaError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"lama_b200 error {code}: {msg}")
        self.code = code


class DeviceOptions(C.Structure):
    _fields_ = [("device", C.c_int32), ("dir_dim", C.c_int32), ("pool_slots", C.c_int32), ("max_beams", C.c_int32), ("timing", C.c_int32),
                ("stream", C.c_uint64)]


class PFOptions(C.Structure):
    _fields_ = [("particles", C.c_uint32), ("srr", C.c_double), ("str", C.c_double), ("stt", C.c_double), ("srt", C.c_double),
                ("meas_sigma", C.c_double), ("meas_sigma_gain", C.c_double), ("trans_thresh", C.c_double), ("rot_thresh", C.c_double),
                ("l2_max", C.c_double), ("truncated_ray", C.c_double), ("truncated_range", C.c_double), ("resolution", C.c_double),
                ("patch_size", C.c_uint32), ("max_iter", C.c_uint32), ("strategy", C.c_int32), ("threads", C.c_int32), ("seed", C.c_uint32),
                ("shard_rank", C.c_uint32), ("shard_count", C.c_uint32), ("dev", DeviceOptions)]


class SlamOptions(C.Structure):
    _fields_ = [("trans_thresh", C.c_double), ("rot_thresh", C.c_double), ("l2_max", C.c_double), ("truncated_ray", C.c_double),
                ("truncated_range", C.c_double), ("resolution", C.c_double), ("patch_size", C.c_uint32), ("max_iter", C.c_uint32),
                ("strategy", C.c_int32), ("occupancy", C.c_int32), ("transient_map", C.c_int32), ("lidar_odometry", C.c_int32),
                ("dev", DeviceOptions)]


class GraphOptions(C.Structure):
    _fields_ = [("slam", SlamOptions), ("key_pose_distance", C.c_double), ("key_pose_angular_distance", C.c_double), ("key_pose_head_delay", C.c_int32),
                ("loop_search_max_distance", C.c_double), ("loop_search_min_distance", C.c_double), ("loop_max_candidates", C.c_int32),
                ("loop_closure_scan_rmse", C.c_double), ("loop_closure_max_candidates", C.c_int32), ("ignore_n_chain_poses", C.c_int32)]


class LocOptions(C.Structure):
    _fields_ = [("trans_thresh", C.c_double), ("rot_thresh", C.c_double), ("l2_max", C.c_double), ("resolution", C.c_double),
                ("patch_size", C.c_uint32), ("max_iter", C.c_uint32), ("strategy", C.c_int32), ("gloc_particles", C.c_uint32),
                ("gloc_iters", C.c_uint32), ("gloc_thresh", C.c_double), ("cov_blend", C.c_double), ("center_xy", C.c_double * 2),
                ("dev", DeviceOptions)]


# every symbol declared in include/lama_b200.h (tests check the library exports all of them)
EXPORTED_SYMBOLS = [
    "lama_last_error", "lama_version", "lama_device_count",
    "lama_pf_options_default", "lama_pf_create", "lama_pf_destroy", "lama_pf_set_prior", "lama_pf_update", "lama_pf_get_pose",
    "lama_pf_stage_scans", "lama_pf_update_staged", "lama_pf_get_traffic",
    "lama_pf_get_best_particle", "lama_pf_get_neff", "lama_pf_get_particles", "lama_pf_get_trajectory", "lama_pf_get_last_resample", "lama_pf_get_resample_digest", "lama_pf_get_summary", "lama_pf_get_memory_usage", "lama_pf_get_timestamps", "lama_shard_unique_id", "lama_pf_shard_connect", "lama_pf_shard_stats", "lama_pgo_optimize", "lama_loop_closure_candidates", "lama_slam_correlate_candidate_scan", "lama_dm_correlate_candidate_scan", "lama_slam_coarse_correlate_candidate_scan", "lama_dm_coarse_correlate_candidate_scan", "lama_dm_match_error",
    "lama_pf_get_counters", "lama_pf_kernel_times", "lama_pf_map_bounds", "lama_pf_get_window", "lama_pf_export_occupancy", "lama_pf_export_distance",
    "lama_pf_shard_begin", "lama_pf_shard_finish", "lama_pf_shard_apply", "lama_pf_shard_apply_local", "lama_pf_shard_map_update",
    "lama_pf_particle_pack_size", "lama_pf_particle_pack", "lama_pf_particle_unpack",
    "lama_slam_options_default", "lama_slam_create", "lama_slam_destroy", "lama_slam_set_pose", "lama_slam_update", "lama_slam_get_pose",
    "lama_slam_get_state", "lama_slam_get_processed_cells", "lama_slam_get_counters", "lama_slam_kernel_times", "lama_slam_map_bounds", "lama_slam_get_window",
    "lama_slam_export_occupancy", "lama_slam_export_distance", "lama_slam_export_logodds",
    "lama_loc_options_default", "lama_loc_create", "lama_loc_destroy", "lama_loc_distance_map", "lama_loc_set_pose", "lama_loc_update",
    "lama_loc_get_pose", "lama_loc_get_state", "lama_loc_get_covar", "lama_loc_get_rmse", "lama_loc_get_solve_stats",
    "lama_pf_distance", "lama_slam_distance", "lama_pf_occupancy_query", "lama_slam_occupancy_query", "lama_w2m", "lama_slam_get_map_stats", "lama_pf_write_map", "lama_pf_export_image", "lama_slam_write_map", "lama_slam_export_image", "lama_dm_write", "lama_dm_read",
    "lama_dm_export_image", "lama_loc_occupancy_read",
    "lama_loc_occupancy_set", "lama_loc_set_seed", "lama_loc_trigger_global_localization", "lama_loc_global_localization_active",
    "lama_dm_create", "lama_dm_destroy", "lama_dm_max_sqdist", "lama_dm_add_obstacles", "lama_dm_remove_obstacles", "lama_dm_update",
    "lama_dm_distance", "lama_dm_bounds", "lama_dm_export", "lama_dm_import", "lama_dm_match_normal_equations", "lama_dm_match_solve",
    "lama_dm_set_follow", "lama_dm_get_window", "lama_dm_get_pool", "lama_dm_kernel_times",
    "lama_pgo_optimize_graph", "lama_graph_options_default", "lama_graph_create", "lama_graph_destroy", "lama_graph_set_pose", "lama_graph_update",
    "lama_graph_get_pose", "lama_graph_get_key_poses", "lama_graph_get_key_cloud", "lama_graph_get_links", "lama_graph_get_last_candidates",
    "lama_graph_get_stats", "lama_graph_slam", "lama_graph_generate_occupancy_map", "lama_graph_generate_coarse_distance_map",
    "lama_om_create", "lama_om_destroy", "lama_om_insert_scans", "lama_om_prune", "lama_om_resolution", "lama_om_bounds", "lama_om_query",
    "lama_om_export", "lama_om_write", "lama_om_export_image", "lama_om_kernel_times", "lama_om_set_follow", "lama_om_get_window", "lama_om_get_pool",
    "lama_tsdm_create", "lama_tsdm_destroy", "lama_tsdm_set_max_distance", "lama_tsdm_max_distance", "lama_tsdm_insert_point_clouds",
    "lama_tsdm_distance", "lama_tsdm_bounds", "lama_tsdm_export", "lama_tsdm_to_mesh", "lama_tsdm_write_ply", "lama_tsdm_kernel_times",
    "lama_om3_create", "lama_om3_destroy", "lama_om3_insert_point_clouds", "lama_om3_apply", "lama_om3_query", "lama_om3_prune",
    "lama_om3_bounds", "lama_om3_export", "lama_om3_write", "lama_om3_read", "lama_om3_export_image", "lama_om3_kernel_times", "lama_w2m3",
    "lama_dm3_create", "lama_dm3_destroy", "lama_dm3_max_sqdist", "lama_dm3_max_distance", "lama_dm3_add_obstacles", "lama_dm3_remove_obstacles",
    "lama_dm3_update", "lama_dm3_distance", "lama_dm3_cell_distance", "lama_dm3_bounds", "lama_dm3_export", "lama_dm3_write", "lama_dm3_read",
    "lama_dm3_export_image", "lama_dm3_kernel_times", "lama_dm3_run_stats", "lama_om3_insert_point_clouds_dm3",
    "lama_pf_save_state", "lama_pf_load_state", "lama_slam_save_state", "lama_slam_load_state", "lama_checkpoint_last_stats",
    "lama_graph_save_state", "lama_graph_load_state", "lama_pf_save_shard_state", "lama_pf_load_state_sharded",
    "lama_locf_create", "lama_locf_destroy", "lama_locf_distance_map", "lama_locf_occupancy_set", "lama_locf_occupancy_read", "lama_locf_set_pose",
    "lama_locf_set_seed", "lama_locf_trigger_global_localization", "lama_locf_global_localization_active", "lama_locf_update", "lama_locf_get",
]


def lib():
    """Loads liblama_b200.so; raises when the CUDA extension has not been built (no fallback)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                              "(make -C iris_lama_b200/csrc). The lama_b200 hot path has no CPU fallback.")
        L = C.CDLL(LIB_PATH)
        L.lama_last_error.restype = C.c_char_p
        L.lama_version.restype = C.c_char_p
        _lib = L
    return _lib


def _chk(rc):
    if rc != 0:
        raise LamaError(rc, lib().lama_last_error().decode())


def _d(a):
    a = np.ascontiguousarray(a, dtype=np.float64)
    return a, a.ctypes.data_as(c_dp)


def _u32(a):
    a = np.ascontiguousarray(a, dtype=np.uint32)
    return a, a.ctypes.data_as(c_u32p)


def _vp(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


_ID3 = np.zeros(3)
_IDQ = np.array([0.0, 0.0, 0.0, 1.0])
_COUNTER_KEYS = ("evals", "ray_cells", "dm_pops", "detached", "gn_iters", "resampled")


def device_count() -> int:
    return lib().lama_device_count()


def _dm_arrays(w, h):
    return dict(sqdist=np.zeros((h, w), np.uint16), valid=np.zeros((h, w), np.uint8), known=np.zeros((h, w), np.uint8),
                ox=np.zeros((h, w), np.int16), oy=np.zeros((h, w), np.int16), queued=np.zeros((h, w), np.uint8))


def _occ_arrays(w, h):
    return dict(occupied=np.zeros((h, w), np.uint16), visited=np.zeros((h, w), np.uint16), known=np.zeros((h, w), np.uint8))


def _dm_args(o):
    return (_vp(o["sqdist"]), _vp(o["valid"]), _vp(o["known"]), _vp(o["ox"]), _vp(o["oy"]), _vp(o["queued"]))


def _counters(fn, h):
    last = np.zeros(6, np.uint64)
    tot = np.zeros(6, np.uint64)
    _chk(fn(h, _vp(last), _vp(tot)))
    return dict(zip(_COUNTER_KEYS, last.tolist())), dict(zip(_COUNTER_KEYS, tot.tolist()))


def _image(fn, args):
    """(height, width) uint8 array of an export_image entry point; pixel (u, v) of the reference image is out[v, u]"""
    dims = (C.c_int * 2)()
    _chk(fn(*args, None, C.c_size_t(0), dims))
    out = np.zeros((dims[1], dims[0]), np.uint8)
    if out.size:
        _chk(fn(*args, _vp(out), C.c_size_t(out.size), dims))
    return out


def w2m(resolution, pts):
    """Map::w2m (map.h:125-126): world points (n, 3) -> cells (n, 2)"""
    p, pp = _d(pts)
    n = p.size // 3
    out = np.zeros((n, 2), np.uint32)
    _chk(lib().lama_w2m(C.c_double(resolution), pp, C.c_int(n), _vp(out)))
    return out


def w2m3(resolution, pts):
    """Map::w2m (map.h:125-126) on all three axes: world points (n, 3) -> cells (n, 3)"""
    p, pp = _d(pts)
    n = p.size // 3
    out = np.zeros((n, 3), np.uint32)
    _chk(lib().lama_w2m3(C.c_double(resolution), pp, C.c_int(n), _vp(out)))
    return out


def write_png(path, grey):
    """8-bit greyscale PNG of a (height, width) uint8 array (the reference hands the same pixels to stb: image_io.cpp:60-68)"""
    import struct
    import zlib
    grey = np.ascontiguousarray(grey, np.uint8)
    h, w = grey.shape
    raw = b"".join(b"\x00" + grey[r].tobytes() for r in range(h))

    def chunk(tag, data):
        body = tag + data
        return struct.pack(">I", len(data)) + body + struct.pack(">I", zlib.crc32(body) & 0xFFFFFFFF)

    with open(path, "wb") as f:
        f.write(b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 0, 0, 0, 0)) + chunk(b"IDAT", zlib.compress(raw, 6)) + chunk(b"IEND", b""))


def _times(fn, h):
    ms = np.zeros(4)
    ln = np.zeros(5, np.uint64)
    _chk(fn(h, ms.ctypes.data_as(c_dp), _vp(ln)))
    return dict(zip(("match_ms", "raycast_ms", "brushfire_ms", "resample_ms"), ms.tolist())), dict(
        zip(("match", "raycast", "brushfire", "resample", "misc"), ln.tolist()))


def _window(fn, h):
    base = np.zeros(2, np.int32)
    dim = C.c_int32(0)
    counts = np.zeros(3, np.uint64)
    _chk(fn(h, base.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(dim), counts.ctypes.data_as(C.POINTER(C.c_uint64))))
    return dict(base=(int(base[0]), int(base[1])), dim=dim.value, shifts=int(counts[0]), parked=int(counts[1]), restored=int(counts[2]))


def _bounds(fn, args):
    mn = np.zeros(2, np.uint32)
    mx = np.zeros(2, np.uint32)
    n = C.c_int(0)
    _chk(fn(*args, mn.ctypes.data_as(c_u32p), mx.ctypes.data_as(c_u32p), C.byref(n)))
    return n.value, mn, mx


class SimplePGO:
    """lama::SimplePGO (include/lama/simple_pgo.h:43-57): node_list (n x {x, y, rotation}), edge_list [(from, to, xyr)], fixed_list [(node, xyr)]"""

    def __init__(self, node_list, edge_list=(), fixed_list=(), device=0):
        self.node_list = np.array(node_list, dtype=np.float64).reshape(-1, 3).copy()
        self.edge_list = list(edge_list)
        self.fixed_list = list(fixed_list)
        self.device = device
        self.status = None
        self.report = None

    def optimize(self) -> bool:
        """SimplePGO::optimize (src/simple_pgo.cpp:48-105): True on SUCCESS (node_list then holds the optimised poses)"""
        ft = np.ascontiguousarray([[e[0], e[1]] for e in self.edge_list], np.int32).reshape(-1, 2)
        ex = np.ascontiguousarray([e[2] for e in self.edge_list], np.float64).reshape(-1, 3)
        fn = np.ascontiguousarray([f[0] for f in self.fixed_list], np.int32)
        fx = np.ascontiguousarray([f[1] for f in self.fixed_list], np.float64).reshape(-1, 3)
        st = C.c_int(-1)
        rep = np.zeros(6)
        _chk(lib().lama_pgo_optimize(C.c_int(self.device), self.node_list.ctypes.data_as(c_dp), C.c_int(len(self.node_list)), ft.ctypes.data_as(c_i32p),
                                     ex.ctypes.data_as(c_dp), C.c_int(len(ft)), fn.ctypes.data_as(c_i32p), fx.ctypes.data_as(c_dp), C.c_int(len(fn)),
                                     C.byref(st), rep.ctypes.data_as(c_dp)))
        self.status = st.value
        self.report = dict(zip(("iterations", "lambda_tries", "cg_iterations", "initial_error", "final_error", "device_ms"), rep.tolist()))
        return st.value == 0


_REPORT_KEYS = ("iterations", "lambda_tries", "cg_iterations", "initial_error", "final_error", "device_ms")


def diagonal_loss(sigmas):
    """miniSAM DiagonalLoss::Sigmas(sigmas) as the 4-vector loss of pgo_optimize_graph"""
    return (float(sigmas[0]), float(sigmas[1]), float(sigmas[2]), 0.0)


def huber_loss(k):
    """miniSAM HuberLoss::Huber(k) as the 4-vector loss of pgo_optimize_graph"""
    return (1.0, 1.0, 1.0, float(k))


def pgo_optimize_graph(nodes, priors=(), betweens=(), device=0):
    """miniSAM Levenberg-Marquardt over an explicit SE2 factor graph on the device.  nodes (n x 3 xyr), priors [(node, xyr, loss)],
    betweens [(from, to, xyr, loss)], loss = diagonal_loss(sigmas) or huber_loss(k).  Returns (status, nodes after the call -- optimised only on
    SUCCESS --, report dict, list of per-lambda-try accept flags)."""
    x = np.array(nodes, dtype=np.float64).reshape(-1, 3).copy()
    pn = np.ascontiguousarray([p[0] for p in priors], np.int32)
    px = np.ascontiguousarray([p[1] for p in priors], np.float64).reshape(-1, 3)
    pl = np.ascontiguousarray([p[2] for p in priors], np.float64).reshape(-1, 4)
    bf = np.ascontiguousarray([[b[0], b[1]] for b in betweens], np.int32).reshape(-1, 2)
    bx = np.ascontiguousarray([b[2] for b in betweens], np.float64).reshape(-1, 3)
    bl = np.ascontiguousarray([b[3] for b in betweens], np.float64).reshape(-1, 4)
    st, tries = C.c_int(-1), C.c_int(0)
    rep = np.zeros(6)
    acc = np.zeros(4096, np.uint8)
    _chk(lib().lama_pgo_optimize_graph(C.c_int(device), x.ctypes.data_as(c_dp), C.c_int(len(x)), pn.ctypes.data_as(c_i32p), px.ctypes.data_as(c_dp),
                                       pl.ctypes.data_as(c_dp), C.c_int(len(pn)), bf.ctypes.data_as(c_i32p), bx.ctypes.data_as(c_dp), bl.ctypes.data_as(c_dp),
                                       C.c_int(len(bf)), C.byref(st), rep.ctypes.data_as(c_dp), _vp(acc), C.c_int(acc.size), C.byref(tries)))
    return st.value, x, dict(zip(_REPORT_KEYS, rep.tolist())), acc[:min(tries.value, acc.size)].tolist()


def loop_closure_candidates(key_xy, ignore_n_chain_poses, query_xy, radius, max_candidates=5):
    """GraphSlam2D::findLoopClosureCandidates (src/graph_slam2d.cpp:283-313): ids of the key poses near `query_xy`, nearest first"""
    k, kp = _d(key_xy)
    q, qp = _d(query_xy)
    ids = np.zeros(max(1, max_candidates), np.int32)
    n = C.c_int(0)
    _chk(lib().lama_loop_closure_candidates(kp, C.c_int(k.size // 2), C.c_int(ignore_n_chain_poses), qp, C.c_double(radius), C.c_int(max_candidates),
                                            ids.ctypes.data_as(c_i32p), C.byref(n)))
    return ids[:n.value].copy()


def _correlate(fn, h, pts, ref_xyr, cand_xyr, origin, quat, ref_pts=None):
    p, pp = _d(pts); o, op = _d(origin); q, qp = _d(quat); r, rp = _d(ref_xyr); c, cp = _d(cand_xyr)
    out = np.zeros(3)
    rmse = C.c_double(0)
    if ref_pts is None:
        _chk(fn(h, pp, C.c_int(p.size // 3), op, qp, rp, cp, out.ctypes.data_as(c_dp), C.byref(rmse)))
    else:
        a, ap = _d(ref_pts)
        _chk(fn(h, ap, C.c_int(a.size // 3), op, qp, pp, C.c_int(p.size // 3), op, qp, rp, cp, out.ctypes.data_as(c_dp), C.byref(rmse)))
    return out, rmse.value


def shard_unique_id() -> bytes:
    """rank 0: the id (ncclGetUniqueId, 128 bytes) every rank passes to PFSlam2D.shardConnect"""
    buf = (C.c_uint8 * 128)()
    _chk(lib().lama_shard_unique_id(buf))
    return bytes(buf)


# ---- checkpoints ------------------------------------------------------------------------------------------------
CKPT_PFSLAM2D, CKPT_SLAM2D, CKPT_LIDAR_ODOMETRY2D, CKPT_GRAPHSLAM2D = 1, 2, 3, 4   # handle kind in the checkpoint header (u32 at byte 12)
CKPT_PFSLAM2D_SHARD = 5   # one rank's shard of a sharded PFSlam2D (PFSlam2D.saveShardState)


def checkpoint_kind(path) -> tuple:
    """(handle kind, first options word) of a checkpoint file's header -- the particle count of a PFSlam2D checkpoint.  Only the header is
    read here; loading checks the whole file."""
    with open(path, "rb") as f:
        head = f.read(60)
    if len(head) < 36 or head[:8] != b"LAMACKPT":
        raise LamaError(-1, f"{path} is not a checkpoint")
    kind = int.from_bytes(head[12:16], "little")
    body = 40 if int.from_bytes(head[8:12], "little") == 2 else 32   # version 2: the 8-byte parked-entry marker opens the body
    if kind == CKPT_PFSLAM2D_SHARD:   # the particle count follows the 16-byte shard record
        return kind, int.from_bytes(head[body + 16:body + 20], "little")
    return kind, int.from_bytes(head[body:body + 4], "little")


def _load_state(fn, path, device, stream, timing):
    d = DeviceOptions(device=device, dir_dim=0, pool_slots=0, max_beams=0, timing=int(timing), stream=stream)
    h = C.c_void_p()
    _chk(fn(str(path).encode(), C.byref(d), C.byref(h)))
    return h


def checkpoint_stats():
    """what the last saveState / loadState on this thread took: dict of ms and sizes (lama_checkpoint_last_stats)"""
    ms = np.zeros(9)
    sz = np.zeros(3, np.uint64)
    _chk(lib().lama_checkpoint_last_stats(ms.ctypes.data_as(c_dp), _vp(sz)))
    keys = ("count_ms", "compact_ms", "gather_ms", "copy_ms", "create_ms", "tables_ms", "encode_ms", "io_ms", "total_ms")
    out = dict(zip(keys, ms.tolist()))
    out.update(used_slots=int(sz[0]), references=int(sz[1]), file_bytes=int(sz[2]))
    return out


class PFSlam2D:
    """lama::PFSlam2D (include/lama/pf_slam2d.h:187-232)."""

    @staticmethod
    def Options(particles, **kw) -> PFOptions:
        o = PFOptions()
        _chk(lib().lama_pf_options_default(C.byref(o)))
        o.particles = particles
        for k, v in kw.items():
            if k in ("device", "dir_dim", "pool_slots", "max_beams", "timing", "stream"):
                setattr(o.dev, k, v)
            else:
                setattr(o, k, v)
        return o

    def __init__(self, options: PFOptions):
        self.options = options
        self.P = options.particles
        self.h = C.c_void_p()
        _chk(lib().lama_pf_create(C.byref(options), C.byref(self.h)))

    def __del__(self):
        if getattr(self, "h", None) and _lib is not None:
            _lib.lama_pf_destroy(self.h)
            self.h = None

    def setPrior(self, x, y, r):
        a, ap = _d([x, y, r])
        _chk(lib().lama_pf_set_prior(self.h, ap))

    def update(self, pts, odom, timestamp=0.0, origin=_ID3, quat=_IDQ) -> bool:
        p, pp = _d(pts)
        o, op = _d(origin)
        q, qp = _d(quat)
        od, odp = _d(odom)
        did = C.c_int(0)
        _chk(lib().lama_pf_update(self.h, pp, C.c_int(p.size // 3), op, qp, odp, C.c_double(timestamp), C.byref(did)))
        return bool(did.value)

    def stageScans(self, scans):
        """scans: (T, N, 3) float64, copied into device memory once."""
        s, sp = _d(scans)
        _chk(lib().lama_pf_stage_scans(self.h, sp, C.c_int(s.shape[0]), C.c_int(s.shape[1])))

    def updateStaged(self, index, odom, timestamp=0.0, origin=_ID3, quat=_IDQ) -> bool:
        o, op = _d(origin)
        q, qp = _d(quat)
        od, odp = _d(odom)
        did = C.c_int(0)
        _chk(lib().lama_pf_update_staged(self.h, C.c_int(index), op, qp, odp, C.c_double(timestamp), C.byref(did)))
        return bool(did.value)

    def traffic(self, reset=False):
        b = np.zeros(2, np.uint64)
        _chk(lib().lama_pf_get_traffic(self.h, _vp(b), C.c_int(int(reset))))
        return int(b[0]), int(b[1])

    def getPose(self):
        out = np.zeros(3)
        _chk(lib().lama_pf_get_pose(self.h, out.ctypes.data_as(c_dp)))
        return out

    def getBestParticleIdx(self) -> int:
        i = C.c_int(0)
        _chk(lib().lama_pf_get_best_particle(self.h, C.byref(i)))
        return i.value

    def getNeff(self) -> float:
        v = C.c_double(0)
        _chk(lib().lama_pf_get_neff(self.h, C.byref(v)))
        return v.value

    def getParticles(self):
        st = np.zeros((self.P, 4))
        w = np.zeros((self.P, 3))
        _chk(lib().lama_pf_get_particles(self.h, st.ctypes.data_as(c_dp), w.ctypes.data_as(c_dp)))
        return st, w

    def trajectory(self, particle, cap=200000):
        n = C.c_int(0)
        _chk(lib().lama_pf_get_trajectory(self.h, C.c_int(particle), None, C.c_int(0), C.byref(n)))
        out = np.zeros((max(n.value, 1), 3))
        _chk(lib().lama_pf_get_trajectory(self.h, C.c_int(particle), out.ctypes.data_as(c_dp), C.c_int(out.shape[0]), C.byref(n)))
        return out[:n.value]

    def lastResample(self):
        idx = np.zeros(self.P, np.int32)
        n = C.c_int(0)
        _chk(lib().lama_pf_get_last_resample(self.h, idx.ctypes.data_as(c_i32p), C.byref(n)))
        return idx[:n.value].copy()

    def resampleDigest(self):
        """(number of resamplings so far, FNV-1a hash of the whole resampling history)"""
        d = np.zeros(2, np.uint64)
        _chk(lib().lama_pf_get_resample_digest(self.h, _vp(d)))
        return int(d[0]), int(d[1])

    def summary(self):
        """PFSlam2D::Summary buckets (pf_slam2d.h:88-129) as host wall-clock sums in ms"""
        t = np.zeros(4)
        _chk(lib().lama_pf_get_summary(self.h, t.ctypes.data_as(c_dp)))
        return dict(zip(("sampling", "solve", "normalize", "resample"), t.tolist()))

    def getMemoryUsage(self):
        """getMemoryUsage() and its (occmem, dmmem) overload (pf_slam2d.cpp:151-176): (total, occmem, dmmem) in bytes of the reference's containers"""
        m = np.zeros(3, np.uint64)
        _chk(lib().lama_pf_get_memory_usage(self.h, _vp(m)))
        return int(m[0]), int(m[1]), int(m[2])

    def getTimestamps(self):
        n = C.c_int(0)
        t = np.zeros(4)
        _chk(lib().lama_pf_get_timestamps(self.h, t.ctypes.data_as(c_dp), 4, C.byref(n)))
        return t[:min(n.value, 4)].tolist()

    def counters(self):
        return _counters(lib().lama_pf_get_counters, self.h)

    def kernelTimes(self):
        return _times(lib().lama_pf_kernel_times, self.h)

    def mapBounds(self, particle, kind):
        return _bounds(lib().lama_pf_map_bounds, (self.h, C.c_int(particle), C.c_int(kind)))

    def window(self):
        """The maps' working window: base (patch coordinates), dim (dir_dim), shifts so far, entries parked now, entries restored so far."""
        return _window(lib().lama_pf_get_window, self.h)

    def exportOccupancy(self, particle, x0, y0, w, h):
        o = _occ_arrays(w, h)
        _chk(lib().lama_pf_export_occupancy(self.h, C.c_int(particle), C.c_uint32(x0), C.c_uint32(y0), C.c_int(w), C.c_int(h),
                                            _vp(o["occupied"]), _vp(o["visited"]), _vp(o["known"])))
        return o

    def exportDistance(self, particle, x0, y0, w, h):
        o = _dm_arrays(w, h)
        _chk(lib().lama_pf_export_distance(self.h, C.c_int(particle), C.c_uint32(x0), C.c_uint32(y0), C.c_int(w), C.c_int(h), *_dm_args(o)))
        return o

    def distance(self, particle, pts, grad=True):
        """getDistanceMap(particle)->distance(point, &gradient) for n world points"""
        p, pp = _d(pts)
        n = p.size // 3
        d = np.zeros(n)
        g = np.zeros((n, 3)) if grad else None
        _chk(lib().lama_pf_distance(self.h, C.c_int(particle), pp, C.c_int(n), d.ctypes.data_as(c_dp), g.ctypes.data_as(c_dp) if grad else None))
        return (d, g) if grad else d

    def occupancyQuery(self, particle, cells):
        """(getProbability, flags) of getOccupancyMap(particle) for n cells; flags bit 0 isFree, bit 1 isOccupied, bit 2 isUnknown"""
        c, cp = _u32(cells)
        n = c.size // 2
        prob, flags = np.zeros(n), np.zeros(n, np.uint8)
        _chk(lib().lama_pf_occupancy_query(self.h, C.c_int(particle), cp, C.c_int(n), prob.ctypes.data_as(c_dp), _vp(flags)))
        return prob, flags

    def writeMap(self, particle, kind, path):
        """Map::write of getOccupancyMap(particle) (kind 0) / getDistanceMap(particle) (kind 1): a reference .sdm file"""
        _chk(lib().lama_pf_write_map(self.h, C.c_int(particle), C.c_int(kind), str(path).encode()))

    def exportImage(self, particle, kind):
        return _image(lib().lama_pf_export_image, (self.h, C.c_int(particle), C.c_int(kind)))

    def saveOccImage(self, path):
        """PFSlam2D::saveOccImage (pf_slam2d.cpp:338-342): the best particle's occupancy map as PNG"""
        write_png(path, self.exportImage(self.getBestParticleIdx(), 0))

    # ---- multi-GPU behind update(): NCCL inside the library --------------------------------------------------
    def shardConnect(self, unique_id: bytes):
        """every rank: connect this handle to the others with the 128-byte id rank 0 got from shard_unique_id()"""
        buf = (C.c_uint8 * 128).from_buffer_copy(bytes(unique_id))
        _chk(lib().lama_pf_shard_connect(self.h, buf))

    def shardStats(self):
        """(collectives issued, bytes of particle maps received)"""
        s = np.zeros(2, np.uint64)
        _chk(lib().lama_pf_shard_stats(self.h, _vp(s)))
        return int(s[0]), int(s[1])

    # ---- split-phase calls used by iris_lama_b200.distributed ------------------------------------------
    def shardBegin(self, pts, odom, timestamp=0.0, origin=_ID3, quat=_IDQ):
        p, pp = _d(pts)
        o, op = _d(origin)
        q, qp = _d(quat)
        od, odp = _d(odom)
        did = C.c_int(0)
        n_local = self.P // max(1, self.options.shard_count)
        out = np.zeros((n_local, 5))
        _chk(lib().lama_pf_shard_begin(self.h, pp, C.c_int(p.size // 3), op, qp, odp, C.c_double(timestamp), C.byref(did), out.ctypes.data_as(c_dp)))
        return did.value, out

    def shardFinish(self, all_results):
        a, ap = _d(all_results)
        res = C.c_int(0)
        idx = np.zeros(self.P, np.int32)
        _chk(lib().lama_pf_shard_finish(self.h, ap, C.byref(res), idx.ctypes.data_as(c_i32p)))
        return bool(res.value), idx

    def shardApply(self, idx, local_src=None):
        idx = np.ascontiguousarray(idx, np.int32)
        if local_src is None:
            _chk(lib().lama_pf_shard_apply(self.h, idx.ctypes.data_as(c_i32p)))
        else:
            ls = np.ascontiguousarray(local_src, np.int32)
            _chk(lib().lama_pf_shard_apply_local(self.h, idx.ctypes.data_as(c_i32p), ls.ctypes.data_as(c_i32p)))

    def shardMapUpdate(self):
        _chk(lib().lama_pf_shard_map_update(self.h))

    def packParticle(self, slot) -> np.ndarray:
        n = C.c_size_t(0)
        _chk(lib().lama_pf_particle_pack_size(self.h, C.c_int(slot), C.byref(n)))
        buf = np.zeros(n.value, np.uint8)
        used = C.c_size_t(0)
        _chk(lib().lama_pf_particle_pack(self.h, C.c_int(slot), _vp(buf), C.c_size_t(buf.size), C.byref(used)))
        return buf[:used.value]

    def unpackParticle(self, slot, buf):
        buf = np.ascontiguousarray(buf, np.uint8)
        _chk(lib().lama_pf_particle_unpack(self.h, C.c_int(slot), _vp(buf), C.c_size_t(buf.size)))

    # ---- checkpoints -----------------------------------------------------------------------------------------
    def saveState(self, path):
        """writes the whole session (options, filter state, device maps) to `path`; the handle is not changed"""
        _chk(lib().lama_pf_save_state(self.h, str(path).encode()))

    @classmethod
    def loadState(cls, path, device=0, stream=0, timing=False) -> "PFSlam2D":
        """a PFSlam2D that continues the saved session bit for bit, on `device` / `stream`"""
        h = _load_state(lib().lama_pf_load_state, path, device, stream, timing)
        _, particles = checkpoint_kind(path)
        self = cls.__new__(cls)
        self.h = h
        self.options = cls.Options(particles, device=device, stream=stream, timing=int(timing))
        self.P = particles
        return self

    def saveShardState(self, path):
        """a sharded rank: writes this rank's shard of the session (the shared filter state, this rank's counters and the maps of its
        particles) to `path`; every rank saves its own file.  The handle is not changed."""
        _chk(lib().lama_pf_save_shard_state(self.h, str(path).encode()))

    @classmethod
    def loadStateSharded(cls, paths, shard_rank, shard_count, device=0, stream=0, timing=False) -> "PFSlam2D":
        """rank `shard_rank` of a `shard_count`-rank filter that continues the session saved in `paths`: the complete set of
        saveShardState files of one save (any order, any saved shard count) or one saveState file.  shard_count 1 gives an unsharded
        handle.  At another shard count than the saved one the rank's counters and Summary buckets start at 0."""
        paths = [str(p) for p in ([paths] if isinstance(paths, (str, os.PathLike)) else paths)]
        arr = (C.c_char_p * max(1, len(paths)))(*[p.encode() for p in paths])
        d = DeviceOptions(device=device, dir_dim=0, pool_slots=0, max_beams=0, timing=int(timing), stream=stream)
        h = C.c_void_p()
        _chk(lib().lama_pf_load_state_sharded(arr, C.c_int(len(paths)), C.c_uint32(shard_rank), C.c_uint32(shard_count), C.byref(d), C.byref(h)))
        _, particles = checkpoint_kind(paths[0])
        self = cls.__new__(cls)
        self.h = h
        self.options = cls.Options(particles, device=device, stream=stream, timing=int(timing), shard_rank=shard_rank, shard_count=shard_count)
        self.P = particles
        return self


class Slam2D:
    """lama::Slam2D (include/lama/slam2d.h:128-161)."""

    @staticmethod
    def Options(**kw) -> SlamOptions:
        o = SlamOptions()
        _chk(lib().lama_slam_options_default(C.byref(o)))
        for k, v in kw.items():
            if k in ("device", "dir_dim", "pool_slots", "max_beams", "timing", "stream"):
                setattr(o.dev, k, v)
            else:
                setattr(o, k, v)
        return o

    def __init__(self, options: SlamOptions):
        self.options = options
        self.h = C.c_void_p()
        _chk(lib().lama_slam_create(C.byref(options), C.byref(self.h)))

    def __del__(self):
        if getattr(self, "h", None) and _lib is not None:
            _lib.lama_slam_destroy(self.h)
            self.h = None

    def setPose(self, x, y, r):
        a, ap = _d([x, y, r])
        _chk(lib().lama_slam_set_pose(self.h, ap))

    def update(self, pts, odom=None, timestamp=0.0, origin=_ID3, quat=_IDQ) -> bool:
        p, pp = _d(pts)
        o, op = _d(origin)
        q, qp = _d(quat)
        od, odp = _d(odom) if odom is not None else (None, None)   # LidarOdometry2D mode takes no odometry
        did = C.c_int(0)
        _chk(lib().lama_slam_update(self.h, pp, C.c_int(p.size // 3), op, qp, odp, C.c_double(timestamp), C.byref(did)))
        return bool(did.value)

    def mapStats(self):
        """(map updates so far, patches deleted by the transient map)"""
        s = np.zeros(2, np.uint64)
        _chk(lib().lama_slam_get_map_stats(self.h, _vp(s)))
        return int(s[0]), int(s[1])

    def getPose(self):
        out = np.zeros(3)
        _chk(lib().lama_slam_get_pose(self.h, out.ctypes.data_as(c_dp)))
        return out

    def state(self):
        out = np.zeros(4)
        _chk(lib().lama_slam_get_state(self.h, out.ctypes.data_as(c_dp)))
        return out

    def getNumberOfProcessedCells(self) -> int:
        n = C.c_uint32(0)
        _chk(lib().lama_slam_get_processed_cells(self.h, C.byref(n)))
        return n.value

    def counters(self):
        return _counters(lib().lama_slam_get_counters, self.h)

    def kernelTimes(self):
        return _times(lib().lama_slam_kernel_times, self.h)

    def mapBounds(self, kind):
        return _bounds(lib().lama_slam_map_bounds, (self.h, C.c_int(kind)))

    def window(self):
        """The maps' working window: base (patch coordinates), dim (dir_dim), shifts so far, entries parked now, entries restored so far."""
        return _window(lib().lama_slam_get_window, self.h)

    def exportOccupancy(self, x0, y0, w, h):
        o = _occ_arrays(w, h)
        _chk(lib().lama_slam_export_occupancy(self.h, C.c_uint32(x0), C.c_uint32(y0), C.c_int(w), C.c_int(h), _vp(o["occupied"]),
                                              _vp(o["visited"]), _vp(o["known"])))
        return o

    def exportLogOdds(self, x0, y0, w, h):
        o = dict(prob=np.zeros((h, w), np.float32), known=np.zeros((h, w), np.uint8))
        _chk(lib().lama_slam_export_logodds(self.h, C.c_uint32(x0), C.c_uint32(y0), C.c_int(w), C.c_int(h), _vp(o["prob"]), _vp(o["known"])))
        return o

    def exportDistance(self, x0, y0, w, h):
        o = _dm_arrays(w, h)
        _chk(lib().lama_slam_export_distance(self.h, C.c_uint32(x0), C.c_uint32(y0), C.c_int(w), C.c_int(h), *_dm_args(o)))
        return o

    def distance(self, pts, grad=True):
        p, pp = _d(pts)
        n = p.size // 3
        d = np.zeros(n)
        g = np.zeros((n, 3)) if grad else None
        _chk(lib().lama_slam_distance(self.h, pp, C.c_int(n), d.ctypes.data_as(c_dp), g.ctypes.data_as(c_dp) if grad else None))
        return (d, g) if grad else d

    def occupancyQuery(self, cells):
        c, cp = _u32(cells)
        n = c.size // 2
        prob, flags = np.zeros(n), np.zeros(n, np.uint8)
        _chk(lib().lama_slam_occupancy_query(self.h, cp, C.c_int(n), prob.ctypes.data_as(c_dp), _vp(flags)))
        return prob, flags

    def correlateCandidateScan(self, pts, ref_xyr, cand_xyr, origin=_ID3, quat=_IDQ):
        """GraphSlam2D::correlateCandidateScan (graph_slam2d.cpp:315-355) against this Slam2D's distance map -> (between xyr, rmse)"""
        return _correlate(lib().lama_slam_correlate_candidate_scan, self.h, pts, ref_xyr, cand_xyr, origin, quat)

    def coarseCorrelateCandidateScan(self, ref_pts, pts, ref_xyr, cand_xyr, origin=_ID3, quat=_IDQ):
        """GraphSlam2D::coarseSearchAndCorrelateCandidateScan (graph_slam2d.cpp:357-392) -> (between xyr, rmse)"""
        return _correlate(lib().lama_slam_coarse_correlate_candidate_scan, self.h, pts, ref_xyr, cand_xyr, origin, quat, ref_pts)

    def writeMap(self, kind, path):
        _chk(lib().lama_slam_write_map(self.h, C.c_int(kind), str(path).encode()))

    def exportImage(self, kind):
        return _image(lib().lama_slam_export_image, (self.h, C.c_int(kind)))

    def saveOccImage(self, path):
        write_png(path, self.exportImage(0))

    def saveState(self, path):
        """writes the whole session (options, state, device maps) to `path`; the handle is not changed"""
        _chk(lib().lama_slam_save_state(self.h, str(path).encode()))

    @staticmethod
    def loadState(path, device=0, stream=0, timing=False) -> "Slam2D":
        """the saved Slam2D, continuing bit for bit; a LidarOdometry2D checkpoint comes back as a LidarOdometry2D"""
        h = _load_state(lib().lama_slam_load_state, path, device, stream, timing)
        kind, _ = checkpoint_kind(path)
        lo = kind == CKPT_LIDAR_ODOMETRY2D
        self = (LidarOdometry2D if lo else Slam2D).__new__(LidarOdometry2D if lo else Slam2D)
        self.h = h
        self.options = Slam2D.Options(lidar_odometry=int(lo), device=device, stream=stream, timing=int(timing))
        return self


class LidarOdometry2D(Slam2D):
    """lama::LidarOdometry2D (include/lama/lidar_odometry_2d.h:45-75): scan-to-map odometry over a transient log-odds map."""

    def __init__(self, resolution=0.05, max_iter=100, **dev):
        super().__init__(Slam2D.Options(lidar_odometry=1, resolution=resolution, max_iter=max_iter, **dev))

    def update(self, pts, timestamp=0.0, origin=_ID3, quat=_IDQ) -> bool:
        return super().update(pts, None, timestamp, origin, quat)


class GraphSlam2D:
    """lama::GraphSlam2D (include/lama/graph_slam2d.h:51-173): key-pose graph SLAM with loop closures over a transient-map Slam2D."""

    @staticmethod
    def Options(**kw) -> GraphOptions:
        """the reference defaults; Slam2D fields (and the device knobs) go to .slam, the nine GraphSlam2D fields to the top level"""
        o = GraphOptions()
        _chk(lib().lama_graph_options_default(C.byref(o)))
        for k, v in kw.items():
            if k in ("device", "dir_dim", "pool_slots", "max_beams", "timing", "stream"):
                setattr(o.slam.dev, k, v)
            elif k in dict(SlamOptions._fields_):
                setattr(o.slam, k, v)
            else:
                setattr(o, k, v)
        return o

    def __init__(self, options: GraphOptions = None):
        self.options = options if options is not None else GraphSlam2D.Options()
        self.h = C.c_void_p()
        _chk(lib().lama_graph_create(C.byref(self.options), C.byref(self.h)))

    def __del__(self):
        if getattr(self, "h", None) and _lib is not None:
            _lib.lama_graph_destroy(self.h)
            self.h = None

    def Init(self, x, y, r):
        """GraphSlam2D::Init (graph_slam2d.cpp:118-121)"""
        a, ap = _d([x, y, r])
        _chk(lib().lama_graph_set_pose(self.h, ap))

    def update(self, pts, odom, timestamp=0.0, origin=_ID3, quat=_IDQ) -> bool:
        """GraphSlam2D::update (graph_slam2d.cpp:188-282)"""
        p, pp = _d(pts); o, op = _d(origin); q, qp = _d(quat); od, odp = _d(odom)
        did = C.c_int(0)
        _chk(lib().lama_graph_update(self.h, pp, C.c_int(p.size // 3), op, qp, odp, C.c_double(timestamp), C.byref(did)))
        return bool(did.value)

    def getPose(self):
        """GraphSlam2D::getPose (graph_slam2d.cpp:127-129): correction + slam pose"""
        out = np.zeros(3)
        _chk(lib().lama_graph_get_pose(self.h, out.ctypes.data_as(c_dp)))
        return out

    def keyPoses(self):
        """key_poses as (corrected n x 3, original n x 3, timestamps n)"""
        n = C.c_int(0)
        _chk(lib().lama_graph_get_key_poses(self.h, None, None, None, C.c_int(0), C.byref(n)))
        cor, org, st = np.zeros((n.value, 3)), np.zeros((n.value, 3)), np.zeros(n.value)
        _chk(lib().lama_graph_get_key_poses(self.h, cor.ctypes.data_as(c_dp), org.ctypes.data_as(c_dp), st.ctypes.data_as(c_dp), C.c_int(n.value), C.byref(n)))
        return cor, org, st

    def keyCloud(self, key):
        """the cloud of key pose `key`: (points n x 3, sensor origin, sensor quaternion xyzw)"""
        n = C.c_int(0)
        _chk(lib().lama_graph_get_key_cloud(self.h, C.c_int(key), None, C.c_int(0), None, None, C.byref(n)))
        pts, o, q = np.zeros((n.value, 3)), np.zeros(3), np.zeros(4)
        _chk(lib().lama_graph_get_key_cloud(self.h, C.c_int(key), pts.ctypes.data_as(c_dp), C.c_int(n.value), o.ctypes.data_as(c_dp), q.ctypes.data_as(c_dp),
                                            C.byref(n)))
        return pts, o, q

    def _ids(self, fn, width):
        n = C.c_int(0)
        _chk(fn(self.h, None, C.c_int(0), C.byref(n)))
        out = np.zeros((n.value, width), np.int32)
        if n.value:
            _chk(fn(self.h, out.ctypes.data_as(c_i32p), C.c_int(n.value), C.byref(n)))
        return out

    def links(self):
        """links (graph_slam2d.h:116-117): n x {candidate key, reference key}"""
        return self._ids(lib().lama_graph_get_links, 2)

    def lastCandidates(self):
        """candidate ids of the latest update's loop search, nearest first"""
        return self._ids(lib().lama_graph_get_last_candidates, 1).ravel()

    def stats(self):
        """{key_poses, loop_factors, optimizations, optimizations_ok, last_status, last_report}"""
        c = np.zeros(4, np.uint64)
        st = C.c_int(-1)
        rep = np.zeros(6)
        _chk(lib().lama_graph_get_stats(self.h, _vp(c), C.byref(st), rep.ctypes.data_as(c_dp)))
        out = dict(zip(("key_poses", "loop_factors", "optimizations", "optimizations_ok"), (int(v) for v in c)))
        out.update(last_status=st.value, last_report=dict(zip(_REPORT_KEYS, rep.tolist())))
        return out

    @property
    def slam(self) -> "Slam2D":
        """the inner Slam2D (the public member `slam`), borrowed: its getters, exports and map writers see the local map"""
        s = Slam2D.__new__(Slam2D)
        s.options = self.options.slam
        s.h = C.c_void_p()
        _chk(lib().lama_graph_slam(self.h, C.byref(s.h)))
        s.owner = self        # keeps the graph alive; destroying the borrowed handle is a no-op
        return s

    def generateOccupancyMap(self, full=False) -> "FrequencyOccupancyMap":
        """GraphSlam2D::generateOccupancyMap (graph_slam2d.cpp:131-164).  The map is BORROWED: owned by this graph and replaced in
        place when the graph recreates it (after a pose-graph optimisation), so an earlier returned object sees the newest map."""
        h = C.c_void_p()
        _chk(lib().lama_graph_generate_occupancy_map(self.h, C.c_int(1 if full else 0), C.byref(h)))
        return FrequencyOccupancyMap(handle=h, owner=self)

    def generateCoarseDistanceMap(self) -> "DynamicDistanceMap":
        """GraphSlam2D::generateCoarseDistanceMap (graph_slam2d.cpp:166-186): a borrowed 0.1 m DynamicDistanceMap with a 5 m reach;
        .processed holds its update() return value"""
        h = C.c_void_p()
        n = C.c_uint32(0)
        _chk(lib().lama_graph_generate_coarse_distance_map(self.h, C.byref(h), C.byref(n)))
        dm = DynamicDistanceMap(handle=h, owner=self)
        dm.processed = n.value
        return dm

    # ---- checkpoints -----------------------------------------------------------------------------------------
    def saveState(self, path):
        """writes the whole session (options, inner Slam2D, key poses and clouds, pose graph, device maps) to `path`; the handle is not
        changed"""
        _chk(lib().lama_graph_save_state(self.h, str(path).encode()))

    @classmethod
    def loadState(cls, path, device=0, stream=0, timing=False) -> "GraphSlam2D":
        """a GraphSlam2D that continues the saved session bit for bit, on `device` / `stream`; `.options` (and `.slam.options`) are the
        saved session's, with the device, stream and timing of this call"""
        h = _load_state(lib().lama_graph_load_state, path, device, stream, timing)
        self = cls.__new__(cls)
        self.h = h
        self.options = _graph_options_of_checkpoint(path, device, stream, timing)
        return self


def _graph_options_of_checkpoint(path, device, stream, timing) -> GraphOptions:
    """the graph options and inner Slam2D options at the start of a kind-4 checkpoint's body (DESIGN.md §13); the loader has checked it"""
    with open(path, "rb") as f:
        f.seek(32)
        b = f.read(56 + 78)
    o = GraphSlam2D.Options()
    (o.key_pose_distance, o.key_pose_angular_distance, o.key_pose_head_delay, o.loop_search_max_distance, o.loop_search_min_distance,
     o.loop_max_candidates, o.loop_closure_scan_rmse, o.loop_closure_max_candidates, o.ignore_n_chain_poses) = struct.unpack_from("<ddiddidii", b)
    s = o.slam
    (s.trans_thresh, s.rot_thresh, s.l2_max, s.truncated_ray, s.truncated_range, s.resolution, s.patch_size, s.max_iter, s.strategy,
     s.occupancy, s.transient_map, s.lidar_odometry, s.dev.dir_dim, s.dev.pool_slots, s.dev.max_beams) = struct.unpack_from("<6dIIii2B3i", b, 56)
    s.dev.device, s.dev.stream, s.dev.timing = device, stream, int(timing)
    return o


class FrequencyOccupancyMap:
    """Device-resident lama::FrequencyOccupancyMap (include/lama/sdm/frequency_occupancy_map.h), stand-alone or borrowed from a
    GraphSlam2D (handle= / owner=, as DynamicDistanceMap).  follow=True: every insertScans moves the directory window over its scans
    group by group instead of failing at the window's edge, and with pool_slots 0 the pool grows (lama_om_set_follow).  A GraphSlam2D's
    map always follows."""

    def __init__(self, resolution=0.05, patch_size=32, center=(0.0, 0.0), handle=None, owner=None, follow=False, **dev):
        self.owner = owner
        if handle is not None:
            self.h = handle
            self.owned = False
            return
        d = DeviceOptions(device=0, dir_dim=64, pool_slots=0, max_beams=2048, timing=0, stream=0)
        for k, v in dev.items():
            setattr(d, k, v)
        c, cp = _d(center)
        self.h = C.c_void_p()
        self.owned = True
        _chk(lib().lama_om_create(C.c_double(resolution), C.c_uint32(patch_size), cp, C.byref(d), C.byref(self.h)))
        if follow:
            _chk(lib().lama_om_set_follow(self.h, C.c_int(1)))

    def __del__(self):
        if getattr(self, "owned", False) and getattr(self, "h", None) and _lib is not None:
            _lib.lama_om_destroy(self.h)
            self.h = None

    @property
    def resolution(self) -> float:
        r = C.c_double(0)
        _chk(lib().lama_om_resolution(self.h, C.byref(r)))
        return r.value

    def insertScans(self, scans, states, full=True, origins=None, quats=None) -> int:
        """the loop of generateOccupancyMap (graph_slam2d.cpp:135-160) for posed scans: `scans` a list of (n_k, 3) clouds, `states`
        (S, 4) SE2 {cos, sin, x, y}, origins (S, 3) / quats (S, 4) xyzw or None (identity).  Returns the number of cell updates."""
        scans = [np.ascontiguousarray(s, np.float64).reshape(-1, 3) for s in scans]
        offsets = np.zeros(len(scans) + 1, np.int64)
        offsets[1:] = np.cumsum([len(s) for s in scans])
        p, pp = _d(np.concatenate(scans) if scans else np.zeros((0, 3)))
        s, sp = _d(np.asarray(states, np.float64).reshape(-1, 4))
        o, op = (None, None) if origins is None else _d(np.asarray(origins, np.float64).reshape(-1, 3))
        q, qp = (None, None) if quats is None else _d(np.asarray(quats, np.float64).reshape(-1, 4))
        cells = C.c_uint64(0)
        _chk(lib().lama_om_insert_scans(self.h, pp, offsets.ctypes.data_as(C.POINTER(C.c_int64)), C.c_int(len(scans)), op, qp, sp,
                                        C.c_int(1 if full else 0), C.byref(cells)))
        return cells.value

    def prune(self):
        """FrequencyOccupancyMap::prune (frequency_occupancy_map.cpp:149-158)"""
        _chk(lib().lama_om_prune(self.h))

    def bounds(self):
        return _bounds(lib().lama_om_bounds, (self.h,))

    def export(self, x0, y0, w, h):
        o = _occ_arrays(w, h)
        _chk(lib().lama_om_export(self.h, C.c_uint32(x0), C.c_uint32(y0), C.c_int(w), C.c_int(h), _vp(o["occupied"]), _vp(o["visited"]), _vp(o["known"])))
        return o

    def query(self, cells):
        """(getProbability, flags bit 0 isFree / bit 1 isOccupied / bit 2 isUnknown) of cells (n, 2)"""
        c, cp = _u32(cells)
        n = c.size // 2
        prob, flags = np.zeros(n), np.zeros(n, np.uint8)
        _chk(lib().lama_om_query(self.h, cp, C.c_int(n), prob.ctypes.data_as(c_dp), _vp(flags)))
        return prob, flags

    def write(self, path):
        """Map::write (map.cpp:490-529): a reference .sdm file"""
        _chk(lib().lama_om_write(self.h, str(path).encode()))

    def exportImage(self):
        return _image(lib().lama_om_export_image, (self.h,))

    def saveImage(self, path):
        write_png(path, self.exportImage())

    def kernelTimes(self):
        return _times(lib().lama_om_kernel_times, self.h)

    def window(self):
        """The working window: base (patch coordinates), dim (dir_dim), shifts so far, entries parked now, entries restored so far."""
        return _window(lib().lama_om_get_window, self.h)

    def pool(self):
        """(pool slots, slots in use)"""
        out = np.zeros(2, np.uint64)
        _chk(lib().lama_om_get_pool(self.h, _vp(out)))
        return int(out[0]), int(out[1])


def _clouds(clouds):
    clouds = [np.ascontiguousarray(c, np.float64).reshape(-1, 3) for c in clouds]
    offsets = np.zeros(len(clouds) + 1, np.int64)
    offsets[1:] = np.cumsum([len(c) for c in clouds])
    return np.ascontiguousarray(np.concatenate(clouds) if clouds else np.zeros((0, 3))), offsets


class _Map3D:
    """What the device-resident 3-D maps share: device options and the handle's lifetime, cells from world points, bounds, box
    shapes and kernel times.  The C-ABI functions are lama_<_PREFIX>_*; _TIMES are the keys of kernelTimes."""

    _PREFIX = None
    _TIMES = ()

    def __init__(self, resolution, patch_size, arg, center, window, dev):
        """lama_<_PREFIX>_create(resolution, patch_size, arg, center, window, dev): arg is the map's own ctypes argument"""
        d = DeviceOptions(device=0, dir_dim=64, pool_slots=0, max_beams=2048, timing=0, stream=0)
        for k, v in dev.items():
            setattr(d, k, v)
        c, cp = _d(center)
        win = None if window is None else (C.c_int32 * 3)(*[int(x) for x in window])
        self.resolution = float(resolution)
        self.h = C.c_void_p()
        _chk(self._fn("create")(C.c_double(resolution), C.c_uint32(patch_size), arg, cp, win, C.byref(d), C.byref(self.h)))

    def __del__(self):
        if getattr(self, "h", None) and _lib is not None:
            getattr(_lib, "lama_%s_destroy" % self._PREFIX)(self.h)
            self.h = None

    def _fn(self, name):
        return getattr(lib(), "lama_%s_%s" % (self._PREFIX, name))

    def _cells(self, cells):
        a = np.asarray(cells)
        if np.issubdtype(a.dtype, np.floating):
            return np.ascontiguousarray(w2m3(self.resolution, a.reshape(-1, 3)))
        return np.ascontiguousarray(a, np.uint32).reshape(-1, 3)

    @staticmethod
    def _box(lo, size):
        """the C arguments of the box lo + [0, size) and the shape of its planes, (size z, size y, size x)"""
        lo = np.ascontiguousarray(lo, np.uint32)
        sz = np.ascontiguousarray(size, np.int32)
        return lo, sz, (int(sz[2]), int(sz[1]), int(sz[0]))

    def bounds(self):
        """(allocated patches, min cell (3,), max cell (3,)) as Map::bounds"""
        mn, mx, n = np.zeros(3, np.uint32), np.zeros(3, np.uint32), C.c_int(0)
        _chk(self._fn("bounds")(self.h, mn.ctypes.data_as(c_u32p), mx.ctypes.data_as(c_u32p), C.byref(n)))
        return n.value, mn, mx

    def kernelTimes(self):
        ms, ln = np.zeros(3), np.zeros(3, np.uint64)
        _chk(self._fn("kernel_times")(self.h, ms.ctypes.data_as(c_dp), _vp(ln)))
        return dict(zip(self._TIMES, ms.tolist())), dict(zip(self._TIMES, ln.tolist()))


class _SdmMap3D(_Map3D):
    """a 3-D map with .sdm files and z-slice images (the TSDM has neither)"""

    def write(self, path):
        """Map::write (map.cpp:490-529): a 3-D .sdm file"""
        _chk(self._fn("write")(self.h, str(path).encode()))

    def read(self, path):
        """Map::read (map.cpp:531-575) into this (empty) map, which takes the file's resolution (map.cpp:548)"""
        _chk(self._fn("read")(self.h, str(path).encode()))
        with open(path, "rb") as f:   # IOHeader.resolution (map.h:95-103), a float at byte 24
            self.resolution = float(np.frombuffer(f.read(28)[24:28], np.float32)[0])

    def exportImage(self, zed=0.0):
        """the z-slice image of sdm::export_to_png(map, file, zed) (export.cpp:46-96), (height, width) uint8"""
        return _image(self._fn("export_image"), (self.h, C.c_double(zed)))

    def saveImage(self, path, zed=0.0):
        write_png(path, self.exportImage(zed))


class TruncatedSignedDistanceMap(_Map3D):
    """Device-resident lama::TruncatedSignedDistanceMap (include/lama/sdm/truncated_signed_distance_map.h).  `window` = patches per
    axis (None: dir_dim x dir_dim x 1 in 2-D, 8 x 8 x 4 in 3-D), centred on `center`."""

    _PREFIX = "tsdm"
    _TIMES = ("insert", "distance", "mesh")

    def __init__(self, resolution, patch_size=32, is3d=False, center=(0.0, 0.0, 0.0), window=None, **dev):
        self.is3d = bool(is3d)
        super().__init__(resolution, patch_size, C.c_int(1 if is3d else 0), center, window, dev)

    def setMaxDistance(self, distance):
        _chk(lib().lama_tsdm_set_max_distance(self.h, C.c_double(distance)))

    def maxDistance(self) -> float:
        r = C.c_double(0)
        _chk(lib().lama_tsdm_max_distance(self.h, C.byref(r)))
        return r.value

    def insertPointClouds(self, clouds, origins=None, quats=None):
        """insertPointCloud on each (n_k, 3) cloud in order; origins (S, 3) / quats (S, 4) xyzw world sensor poses or None (zero /
        identity).  Returns the (S,) return values: distinct hit cells per cloud."""
        p, offsets = _clouds(clouds)
        o = None if origins is None else np.ascontiguousarray(origins, np.float64).reshape(-1, 3)
        q = None if quats is None else np.ascontiguousarray(quats, np.float64).reshape(-1, 4)
        out = np.zeros(len(offsets) - 1, np.uint64)
        _chk(lib().lama_tsdm_insert_point_clouds(self.h, _vp(p), offsets.ctypes.data_as(C.POINTER(C.c_int64)), C.c_int(len(offsets) - 1), _vp(o), _vp(q),
                                                 _vp(out)))
        return out

    def insertPointCloud(self, points, origin=None, quat=None) -> int:
        """insertPointCloud (truncated_signed_distance_map.cpp:141-158)"""
        return int(self.insertPointClouds([points], None if origin is None else [origin], None if quat is None else [quat])[0])

    def distance(self, points, gradient=False):
        """distance(Vector3d, gradient) of (n, 3) world points: (n,) distances, and (n, 3) gradients with gradient=True"""
        p, pp = _d(np.asarray(points, np.float64).reshape(-1, 3))
        n = p.size // 3
        dist, grad = np.zeros(n), np.zeros((n, 3))
        _chk(lib().lama_tsdm_distance(self.h, pp, C.c_int(n), dist.ctypes.data_as(c_dp), grad.ctypes.data_as(c_dp) if gradient else None))
        return (dist, grad) if gradient else dist

    def export(self, lo, size):
        """cells of the box lo + [0, size): dict(distance, weight, on) shaped (size z, size y, size x)"""
        lo, sz, shape = self._box(lo, size)
        o = dict(distance=np.zeros(shape, np.float32), weight=np.zeros(shape, np.float32), on=np.zeros(shape, np.uint8))
        _chk(lib().lama_tsdm_export(self.h, _vp(lo), _vp(sz), _vp(o["distance"]), _vp(o["weight"]), _vp(o["on"])))
        return o

    def toMesh(self):
        """toMesh (:220-272): (vertices (n, 3) float32, index (n,) uint32 = 0..n-1), 3 vertices per triangle"""
        n = C.c_size_t(0)
        _chk(lib().lama_tsdm_to_mesh(self.h, None, C.c_size_t(0), C.byref(n)))
        v = np.zeros((n.value, 3), np.float32)
        if n.value:
            _chk(lib().lama_tsdm_to_mesh(self.h, _vp(v), C.c_size_t(n.value), C.byref(n)))
        return v, np.arange(n.value, dtype=np.uint32)


class OccupancyMap3D(_SdmMap3D):
    """Device-resident lama::FrequencyOccupancyMap (kind="frequency") or lama::ProbabilisticOccupancyMap (kind="logodds") with
    is3d = true (include/lama/sdm/*_occupancy_map.h).  `window` = patches per axis (None: 8 x 8 x 4), centred on `center`.

    Cells are (n, 3) integer map coordinates; floating-point arrays are world points and go through Map::w2m (w2m3), as the
    reference's Vector3d overloads do."""

    KINDS = {"frequency": 0, "logodds": 1}
    SET_FREE, SET_OCCUPIED, SET_UNKNOWN = 0, 1, 2
    _PREFIX = "om3"
    _TIMES = ("insert", "apply", "query")

    def __init__(self, resolution, kind="frequency", patch_size=32, center=(0.0, 0.0, 0.0), window=None, **dev):
        self.kind = kind
        super().__init__(resolution, patch_size, C.c_int(self.KINDS[kind]), center, window, dev)

    def insertPointClouds(self, clouds, origins=None, quats=None, full=True) -> int:
        """generateOccupancyMap's loop body (graph_slam2d.cpp:146-158) for every point of every (n_k, 3) cloud in order: setOccupied
        of the hit and, with full, setFree along the ray from the sensor origin.  origins (S, 3) / quats (S, 4) xyzw world sensor poses
        or None (zero / identity).  Returns the number of cell updates."""
        p, offsets = _clouds(clouds)
        o = None if origins is None else np.ascontiguousarray(origins, np.float64).reshape(-1, 3)
        q = None if quats is None else np.ascontiguousarray(quats, np.float64).reshape(-1, 4)
        n = C.c_uint64(0)
        _chk(lib().lama_om3_insert_point_clouds(self.h, _vp(p), offsets.ctypes.data_as(C.POINTER(C.c_int64)), C.c_int(len(offsets) - 1), _vp(o), _vp(q),
                                                C.c_int(1 if full else 0), C.byref(n)))
        return n.value

    def updateMaps(self, distance_map, clouds, origins=None, quats=None, full=True, counts=False):
        """insertPointClouds with the DynamicDistanceMap3D `distance_map` kept in step, as the reference's map update (slam2d.cpp:271-316):
        a setOccupied that returns true is an addObstacle, a setFree that returns true a removeObstacle, and distance_map.update() runs
        after every cloud.  Both maps must share device, resolution and window.  Returns (cell updates, processed (S,) uint32, every
        cloud's update()), and with counts also {"events", "pushes"}: the setter calls that returned true, and those whose distance-map
        op pushed a heap entry."""
        p, offsets = _clouds(clouds)
        o = None if origins is None else np.ascontiguousarray(origins, np.float64).reshape(-1, 3)
        q = None if quats is None else np.ascontiguousarray(quats, np.float64).reshape(-1, 4)
        n = C.c_uint64(0)
        processed = np.zeros(len(offsets) - 1, np.uint32)
        cnt = np.zeros(2, np.uint64)
        _chk(lib().lama_om3_insert_point_clouds_dm3(self.h, distance_map.h, _vp(p), offsets.ctypes.data_as(C.POINTER(C.c_int64)), C.c_int(len(offsets) - 1),
                                                    _vp(o), _vp(q), C.c_int(1 if full else 0), C.byref(n), _vp(processed), _vp(cnt)))
        if counts:
            return n.value, processed, dict(events=int(cnt[0]), pushes=int(cnt[1]))
        return n.value, processed

    def apply(self, cells, ops):
        """the setters in list order: ops (n,) of SET_FREE / SET_OCCUPIED / SET_UNKNOWN.  Returns what each call returns, (n,) bool."""
        c = self._cells(cells)
        o = np.ascontiguousarray(np.broadcast_to(np.asarray(ops, np.uint8), (len(c),)))
        changed = np.zeros(len(c), np.uint8)
        _chk(lib().lama_om3_apply(self.h, _vp(c), _vp(o), C.c_int(len(c)), _vp(changed)))
        return changed.astype(bool)

    def setFree(self, cells):
        return self.apply(cells, self.SET_FREE)

    def setOccupied(self, cells):
        return self.apply(cells, self.SET_OCCUPIED)

    def setUnknown(self, cells):
        return self.apply(cells, self.SET_UNKNOWN)

    def query(self, cells):
        """(getProbability (n,), flags (n,) bit 0 isFree / bit 1 isOccupied / bit 2 isUnknown)"""
        c = self._cells(cells)
        prob, flags = np.zeros(len(c)), np.zeros(len(c), np.uint8)
        _chk(lib().lama_om3_query(self.h, _vp(c), C.c_int(len(c)), prob.ctypes.data_as(c_dp), _vp(flags)))
        return prob, flags

    def getProbability(self, cells):
        return self.query(cells)[0]

    def isFree(self, cells):
        return (self.query(cells)[1] & 1) != 0

    def isOccupied(self, cells):
        return (self.query(cells)[1] & 2) != 0

    def isUnknown(self, cells):
        return (self.query(cells)[1] & 4) != 0

    def prune(self):
        """FrequencyOccupancyMap::prune (frequency_occupancy_map.cpp:149-158)"""
        _chk(lib().lama_om3_prune(self.h))

    def export(self, lo, size):
        """cells of the box lo + [0, size), shaped (size z, size y, size x): dict(occupied, visited, known) for a frequency map,
        dict(prob (float32 log-odds), known) for a log-odds map, and `word`, the raw 32-bit cells"""
        lo, sz, shape = self._box(lo, size)
        w, k = np.zeros(shape, np.uint32), np.zeros(shape, np.uint8)
        _chk(lib().lama_om3_export(self.h, _vp(lo), _vp(sz), _vp(w), _vp(k)))
        if self.kind == "frequency":
            return dict(word=w, occupied=(w & 0xFFFF).astype(np.uint16), visited=(w >> 16).astype(np.uint16), known=k)
        return dict(word=w, prob=w.view(np.float32), known=k)


class DynamicDistanceMap3D(_SdmMap3D):
    """Device-resident lama::DynamicDistanceMap with is3d = true (include/lama/sdm/dynamic_distance_map.h): the six-neighbour dynamic
    brushfire.  setMaxDistance is fixed at creation (`l2_max`); `window` = patches per axis (None: 8 x 8 x 4), centred on `center`.

    Cells are (n, 3) integer map coordinates; floating-point arrays passed as cells are world points and go through Map::w2m
    (w2m3), as the reference's Vector3d overloads do.  addObstacle / removeObstacle are queued and applied, in order, by update()
    or by the next read of the map, which also takes the file's max_sqdist (readParameters)."""

    _PREFIX = "dm3"
    _TIMES = ("update", "distance", "cells")

    def __init__(self, resolution, l2_max=0.5, patch_size=32, center=(0.0, 0.0, 0.0), window=None, **dev):
        super().__init__(resolution, patch_size, C.c_double(l2_max), center, window, dev)

    @property
    def max_sqdist(self):
        v = C.c_uint32(0)
        _chk(lib().lama_dm3_max_sqdist(self.h, C.byref(v)))
        return v.value

    def maxDistance(self):
        """maxDistance (dynamic_distance_map.cpp:155-158)"""
        v = C.c_double(0)
        _chk(lib().lama_dm3_max_distance(self.h, C.byref(v)))
        return v.value

    def addObstacle(self, cells):
        """addObstacle (:212-226) of every cell, in order"""
        c = self._cells(cells)
        _chk(lib().lama_dm3_add_obstacles(self.h, _vp(c), C.c_int(len(c))))

    def removeObstacle(self, cells):
        """removeObstacle (:228-242) of every cell, in order"""
        c = self._cells(cells)
        _chk(lib().lama_dm3_remove_obstacles(self.h, _vp(c), C.c_int(len(c))))

    def update(self) -> int:
        """update() (:160-197): the number of processed cells"""
        n = C.c_uint32(0)
        _chk(lib().lama_dm3_update(self.h, C.byref(n)))
        return n.value

    def distance(self, pts, grad=True):
        """distance(Vector3d, gradient) (:93-133) of world points (n, 3): distances (n,) and, with grad, gradients (n, 3)"""
        p, pp = _d(pts)
        n = p.size // 3
        d = np.zeros(n)
        g = np.zeros((n, 3)) if grad else None
        _chk(lib().lama_dm3_distance(self.h, pp, C.c_int(n), d.ctypes.data_as(c_dp), g.ctypes.data_as(c_dp) if grad else None))
        return (d, g) if grad else d

    def cellDistance(self, cells):
        """distance(Vector3ui) (:140-147) of integer cells (n, 3)"""
        c = np.ascontiguousarray(cells, np.uint32).reshape(-1, 3)
        d = np.zeros(len(c))
        _chk(lib().lama_dm3_cell_distance(self.h, _vp(c), C.c_int(len(c)), d.ctypes.data_as(c_dp)))
        return d

    def export(self, lo, size):
        """cells of the box lo + [0, size), shaped (size z, size y, size x): dict(word (raw uint64), sqdist, ox, oy, oz, valid, queued,
        known)"""
        lo, sz, shape = self._box(lo, size)
        w, k = np.zeros(shape, np.uint64), np.zeros(shape, np.uint8)
        _chk(lib().lama_dm3_export(self.h, _vp(lo), _vp(sz), _vp(w), _vp(k)))
        return dm3_fields(w, k)

    def runStats(self):
        """{launches, grows, raise_cap, lower_cap} of the brushfire since creation"""
        s = np.zeros(4, np.uint64)
        _chk(lib().lama_dm3_run_stats(self.h, _vp(s)))
        return dict(zip(("launches", "grows", "raise_cap", "lower_cap"), s.tolist()))


def dm3_fields(words, known):
    """the fields of 64-bit 3-D distance cells (lama_dm3_export's layout)"""
    w = np.asarray(words, np.uint64)
    b = w.view(np.uint8).reshape(w.shape + (8,))
    return dict(word=w, ox=b[..., 0].view(np.int8).astype(np.int16), oy=b[..., 1].view(np.int8).astype(np.int16),
                oz=b[..., 2].view(np.int8).astype(np.int16), valid=(b[..., 3] & 1), queued=(b[..., 3] >> 1) & 1,
                sqdist=(w >> np.uint64(32)).astype(np.uint16), known=np.asarray(known, np.uint8))


class DynamicDistanceMap:
    """Device-resident lama::DynamicDistanceMap (include/lama/sdm/dynamic_distance_map.h:55-66).  follow=True (setFollow): read()
    loads a file of any size and update() moves the directory window over its obstacles instead of failing at the window's edge, and
    with pool_slots 0 the pool grows (lama_dm_set_follow).  A Loc2D follows exactly when its distance_map does."""

    def __init__(self, resolution=0.05, patch_size=32, l2_max=0.5, center=(0.0, 0.0), handle=None, owner=None, follow=False, **dev):
        self.owner = owner
        if handle is not None:
            self.h = handle
            self.owned = False
            return
        d = DeviceOptions(device=0, dir_dim=64, pool_slots=0, max_beams=2048, timing=0, stream=0)
        for k, v in dev.items():
            setattr(d, k, v)
        c, cp = _d(center)
        self.h = C.c_void_p()
        self.owned = True
        _chk(lib().lama_dm_create(C.c_double(resolution), C.c_uint32(patch_size), C.c_double(l2_max), cp, C.byref(d), C.byref(self.h)))
        if follow:
            self.setFollow(True)

    def __del__(self):
        if getattr(self, "owned", False) and getattr(self, "h", None) and _lib is not None:
            _lib.lama_dm_destroy(self.h)
            self.h = None

    @property
    def max_sqdist(self):
        v = C.c_uint32(0)
        _chk(lib().lama_dm_max_sqdist(self.h, C.byref(v)))
        return v.value

    def addObstacle(self, cells):
        c, cp = _u32(cells)
        _chk(lib().lama_dm_add_obstacles(self.h, cp, C.c_int(c.size // 2)))

    def removeObstacle(self, cells):
        c, cp = _u32(cells)
        _chk(lib().lama_dm_remove_obstacles(self.h, cp, C.c_int(c.size // 2)))

    def update(self) -> int:
        n = C.c_uint32(0)
        _chk(lib().lama_dm_update(self.h, C.byref(n)))
        return n.value

    def distance(self, pts, grad=True):
        p, pp = _d(pts)
        n = p.size // 3
        d = np.zeros(n)
        g = np.zeros((n, 3)) if grad else None
        _chk(lib().lama_dm_distance(self.h, pp, C.c_int(n), d.ctypes.data_as(c_dp), g.ctypes.data_as(c_dp) if grad else None))
        return (d, g) if grad else d

    def bounds(self):
        return _bounds(lib().lama_dm_bounds, (self.h,))

    def export(self, x0, y0, w, h):
        o = _dm_arrays(w, h)
        _chk(lib().lama_dm_export(self.h, C.c_uint32(x0), C.c_uint32(y0), C.c_int(w), C.c_int(h), *_dm_args(o)))
        return o

    def import_(self, x0, y0, fields):
        h, w = fields["sqdist"].shape
        f = {k: np.ascontiguousarray(fields[k]) for k in ("sqdist", "valid", "known", "ox", "oy", "queued")}
        _chk(lib().lama_dm_import(self.h, C.c_uint32(x0), C.c_uint32(y0), C.c_int(w), C.c_int(h), *_dm_args(f)))

    def write(self, path):
        """Map::write (map.cpp:490-529): a reference .sdm file"""
        _chk(lib().lama_dm_write(self.h, str(path).encode()))

    def read(self, path):
        """Map::read (map.cpp:531-575) into this (empty) map"""
        _chk(lib().lama_dm_read(self.h, str(path).encode()))

    def exportImage(self):
        return _image(lib().lama_dm_export_image, (self.h,))

    def setFollow(self, on=True):
        _chk(lib().lama_dm_set_follow(self.h, C.c_int(1 if on else 0)))

    def window(self):
        """The working window: base (patch coordinates), dim (dir_dim), shifts so far, entries parked now, entries restored so far."""
        return _window(lib().lama_dm_get_window, self.h)

    def pool(self):
        """(pool slots, slots in use)"""
        out = np.zeros(2, np.uint64)
        _chk(lib().lama_dm_get_pool(self.h, _vp(out)))
        return int(out[0]), int(out[1])

    def kernelTimes(self):
        return _times(lib().lama_dm_kernel_times, self.h)

    def matchNormalEquations(self, pts, states, robust=(1, 0.15), meas_sigma=0.05, origin=_ID3, quat=_IDQ):
        p, pp = _d(pts)
        o, op = _d(origin)
        q, qp = _d(quat)
        s, sp = _d(states)
        count = s.size // 4
        out = np.zeros((count, 12))
        _chk(lib().lama_dm_match_normal_equations(self.h, pp, C.c_int(p.size // 3), op, qp, sp, C.c_int(count), C.c_int(robust[0]),
                                                  C.c_double(robust[1]), C.c_double(meas_sigma), out.ctypes.data_as(c_dp)))
        return out

    def matchError(self, pts, states, origin=_ID3, quat=_IDQ):
        """MatchSurface2D::error (match_surface_2d.cpp:92-116) at `count` states"""
        p, pp = _d(pts); o, op = _d(origin); q, qp = _d(quat); s, sp = _d(states)
        count = s.size // 4
        out = np.zeros(count)
        _chk(lib().lama_dm_match_error(self.h, pp, C.c_int(p.size // 3), op, qp, sp, C.c_int(count), out.ctypes.data_as(c_dp)))
        return out

    def correlateCandidateScan(self, pts, ref_xyr, cand_xyr, origin=_ID3, quat=_IDQ):
        return _correlate(lib().lama_dm_correlate_candidate_scan, self.h, pts, ref_xyr, cand_xyr, origin, quat)

    def coarseCorrelateCandidateScan(self, ref_pts, pts, ref_xyr, cand_xyr, origin=_ID3, quat=_IDQ):
        return _correlate(lib().lama_dm_coarse_correlate_candidate_scan, self.h, pts, ref_xyr, cand_xyr, origin, quat, ref_pts)

    def matchSolve(self, pts, states, strategy=0, robust=(1, 0.15), max_iter=100, origin=_ID3, quat=_IDQ):
        p, pp = _d(pts)
        o, op = _d(origin)
        q, qp = _d(quat)
        s = np.array(states, dtype=np.float64).reshape(-1, 4).copy()
        count = s.shape[0]
        stats = np.zeros((count, 2), np.uint32)
        sums = np.zeros((count, 12))
        _chk(lib().lama_dm_match_solve(self.h, pp, C.c_int(p.size // 3), op, qp, s.ctypes.data_as(c_dp), C.c_int(count), C.c_int(strategy),
                                       C.c_int(robust[0]), C.c_double(robust[1]), C.c_uint32(max_iter), stats.ctypes.data_as(c_u32p),
                                       sums.ctypes.data_as(c_dp)))
        return s, stats, sums


class Loc2D:
    """lama::Loc2D match path (include/lama/loc2d.h:103-130)."""

    @staticmethod
    def Options(**kw) -> LocOptions:
        o = LocOptions()
        _chk(lib().lama_loc_options_default(C.byref(o)))
        for k, v in kw.items():
            if k in ("device", "dir_dim", "pool_slots", "max_beams", "timing", "stream"):
                setattr(o.dev, k, v)
            elif k == "center":
                o.center_xy[0], o.center_xy[1] = v
            else:
                setattr(o, k, v)
        return o

    def __init__(self, options: LocOptions):
        self.options = options
        self.h = C.c_void_p()
        _chk(lib().lama_loc_create(C.byref(options), C.byref(self.h)))
        dm = C.c_void_p()
        _chk(lib().lama_loc_distance_map(self.h, C.byref(dm)))
        self.distance_map = DynamicDistanceMap(handle=dm, owner=self)

    def __del__(self):
        if getattr(self, "h", None) and _lib is not None:
            _lib.lama_loc_destroy(self.h)
            self.h = None

    def setPose(self, x, y, r):
        a, ap = _d([x, y, r])
        _chk(lib().lama_loc_set_pose(self.h, ap))

    def update(self, pts, odom, timestamp=0.0, force_update=False, origin=_ID3, quat=_IDQ) -> bool:
        p, pp = _d(pts)
        o, op = _d(origin)
        q, qp = _d(quat)
        od, odp = _d(odom)
        did = C.c_int(0)
        _chk(lib().lama_loc_update(self.h, pp, C.c_int(p.size // 3), op, qp, odp, C.c_double(timestamp), C.c_int(int(force_update)), C.byref(did)))
        return bool(did.value)

    def getPose(self):
        out = np.zeros(3)
        _chk(lib().lama_loc_get_pose(self.h, out.ctypes.data_as(c_dp)))
        return out

    def state(self):
        out = np.zeros(4)
        _chk(lib().lama_loc_get_state(self.h, out.ctypes.data_as(c_dp)))
        return out

    def getCovar(self):
        out = np.zeros((3, 3))
        _chk(lib().lama_loc_get_covar(self.h, out.ctypes.data_as(c_dp)))
        return out

    def getRMSE(self):
        v = C.c_double(0)
        _chk(lib().lama_loc_get_rmse(self.h, C.byref(v)))
        return v.value

    def occupancyRead(self, path):
        """occupancy_map->read(path): a SimpleOccupancyMap .sdm file"""
        _chk(lib().lama_loc_occupancy_read(self.h, str(path).encode()))

    def occupancySet(self, cells, state):
        """public occupancy_map (SimpleOccupancyMap): state -1 setFree, 0 setUnknown, 1 setOccupied"""
        c, cp = _u32(cells)
        _chk(lib().lama_loc_occupancy_set(self.h, cp, C.c_int(c.size // 2), C.c_int(state)))

    def setSeed(self, seed):
        _chk(lib().lama_loc_set_seed(self.h, C.c_uint32(seed)))

    def triggerGlobalLocalization(self):
        _chk(lib().lama_loc_trigger_global_localization(self.h))

    def globalLocalizationActive(self) -> bool:
        a = C.c_int(0)
        _chk(lib().lama_loc_global_localization_active(self.h, C.byref(a)))
        return bool(a.value)

    def solveStats(self):
        s = np.zeros(2, np.uint32)
        _chk(lib().lama_loc_get_solve_stats(self.h, s.ctypes.data_as(c_u32p)))
        return s


def _fleet_update_args(robots, scans, odoms, force=None, origins=None, quats=None):
    """the arrays of lama_locf_update: robot indices, the scans' points back to back (xyz), points per scan, sensor origins (k x 3) and
    quaternions (k x 4, xyzw) or None, odometry (k x 3), force flags or None"""
    rb = np.ascontiguousarray(robots, dtype=np.int32).reshape(-1)
    k = rb.size
    if len(scans) != k:
        raise ValueError("one scan per robot")
    sc = [np.asarray(p, dtype=np.float64).reshape(-1, 3) for p in scans]
    pts = np.ascontiguousarray(np.concatenate(sc) if k else np.zeros((0, 3)))
    n = np.array([p.shape[0] for p in sc], np.int32)
    od = np.ascontiguousarray(odoms, dtype=np.float64).reshape(k, 3)
    fo = None if force is None else np.ascontiguousarray(force, dtype=np.int32).reshape(k)
    org = None if origins is None else np.ascontiguousarray(origins, dtype=np.float64).reshape(k, 3)
    qt = None if quats is None else np.ascontiguousarray(quats, dtype=np.float64).reshape(k, 4)
    return rb, pts, n, org, qt, od, fo


class Loc2DFleet:
    """Many robots localising on one shared map (lama_locf_*).  Robot r gives what a Loc2D with the same options, map and seed gives
    when it is fed only r's calls in the same order.  update() matches every robot of a call in one device launch per step."""

    Options = Loc2D.Options

    def __init__(self, options: LocOptions, robots: int):
        self.options = options
        self.robots = int(robots)
        self.h = C.c_void_p()
        _chk(lib().lama_locf_create(C.byref(options), C.c_int(self.robots), C.byref(self.h)))
        dm = C.c_void_p()
        _chk(lib().lama_locf_distance_map(self.h, C.byref(dm)))
        self.distance_map = DynamicDistanceMap(handle=dm, owner=self)

    def __del__(self):
        if getattr(self, "h", None) and _lib is not None:
            _lib.lama_locf_destroy(self.h)
            self.h = None

    def update(self, robots, scans, odoms, force=None, origins=None, quats=None):
        """robots[k] takes scans[k] (n x 3) with odometry odoms[k] (x, y, rotation); per-robot force flags and sensor origins / quaternions
        (xyzw) are optional.  Returns the did_update flags (bool array, in call order)."""
        rb, pts, n, org, qt, od, fo = _fleet_update_args(robots, scans, odoms, force, origins, quats)
        did = np.zeros(rb.size, np.int32)
        _chk(lib().lama_locf_update(self.h, C.c_int(rb.size), _vp(rb), _vp(pts), _vp(n), _vp(org), _vp(qt), _vp(od), _vp(fo), _vp(did)))
        return did.astype(bool)

    def _get(self):
        st, cov, rmse, stats = np.zeros((self.robots, 4)), np.zeros((self.robots, 3, 3)), np.zeros(self.robots), np.zeros((self.robots, 2), np.uint32)
        _chk(lib().lama_locf_get(self.h, _vp(st), _vp(cov), _vp(rmse), _vp(stats)))
        return st, cov, rmse, stats

    def states(self):
        """(robots, 4): cos, sin, x, y of every robot"""
        return self._get()[0]

    def covars(self):
        return self._get()[1]

    def rmses(self):
        return self._get()[2]

    def solveStats(self):
        """(robots, 2): iterations and residual evaluations of every robot's last tracking match"""
        return self._get()[3]

    def setPose(self, robot, x, y, r):
        a, ap = _d([x, y, r])
        _chk(lib().lama_locf_set_pose(self.h, C.c_int(robot), ap))

    def setSeed(self, robot, seed):
        _chk(lib().lama_locf_set_seed(self.h, C.c_int(robot), C.c_uint32(seed)))

    def triggerGlobalLocalization(self, robot):
        _chk(lib().lama_locf_trigger_global_localization(self.h, C.c_int(robot)))

    def globalLocalizationActive(self, robot) -> bool:
        a = C.c_int(0)
        _chk(lib().lama_locf_global_localization_active(self.h, C.c_int(robot), C.byref(a)))
        return bool(a.value)

    def occupancyRead(self, path):
        """the shared SimpleOccupancyMap from a .sdm file"""
        _chk(lib().lama_locf_occupancy_read(self.h, str(path).encode()))

    def occupancySet(self, cells, state):
        """the shared SimpleOccupancyMap: state -1 setFree, 0 setUnknown, 1 setOccupied"""
        c, cp = _u32(cells)
        _chk(lib().lama_locf_occupancy_set(self.h, cp, C.c_int(c.size // 2), C.c_int(state)))
