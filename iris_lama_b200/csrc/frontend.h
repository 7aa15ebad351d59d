// frontend.h -- host-side mirrors of lama::PFSlam2D / Slam2D / Loc2D on top of the device Engine.
// The orchestration that the reference keeps on its main thread (odometry sampling with the global
// mt19937, weight normalisation, systematic resampling, motion gating) stays on the host in fp64 with
// libstdc++ <random>, so resampling indices are bit-exact with a reference build; the per-particle
// loops the reference farms to its thread pool (src/pf_slam2d.cpp:254-266,292-302) are the kernels.
#pragma once

#include <memory>
#include <random>
#include <unordered_map>
#include <string>
#include <vector>

#include "engine.h"
#include "pgo.h"

namespace lama_b200 {

struct ShardComm;
struct CheckpointStats;
class CkptWriter;
class CkptReader;

struct DeviceOptions {
    int device = 0, dir_dim = 64, pool_slots = 0, max_beams = 2048, timing = 0;
    uint64_t stream = 0;
};

// ---- PFSlam2D ---------------------------------------------------------------------------------------
struct PFOptions {  // include/lama/pf_slam2d.h:132-185
    uint32_t particles = 1;
    double srr = 0.1, str = 0.2, stt = 0.1, srt = 0.2;
    double meas_sigma = 0.05, meas_sigma_gain = 3;
    double trans_thresh = 0.5, rot_thresh = 0.5;
    double l2_max = 0.5;
    double truncated_ray = 0.0, truncated_range = 0.0;
    double resolution = 0.05;
    uint32_t patch_size = 32, max_iter = 100;
    int strategy = 0;
    int threads = -1;
    uint32_t seed = 0;
    uint32_t shard_rank = 0, shard_count = 1;
    DeviceOptions dev;
};

struct Counters {
    uint64_t evals = 0, ray_cells = 0, dm_pops = 0, detached = 0, gn_iters = 0, resampled = 0;
    void add(const Counters& o)
    {
        evals += o.evals; ray_cells += o.ray_cells; dm_pops += o.dm_pops; detached += o.detached; gn_iters += o.gn_iters; resampled += o.resampled;
    }
};

class PFSlam2D {
public:
    static PFSlam2D* create(const PFOptions& o, std::string& err);
    ~PFSlam2D();

    void set_prior(double x, double y, double r) { prior_ = se2_from_xyr(x, y, r); }
    // bool PFSlam2D::update(...)  (src/pf_slam2d.cpp:178-312); returns a LAMA_* status
    int update(const double* pts, int n, const double* origin, const double* quat, const double odom_xyr[3], double stamp, bool* did_update);

    // Scans resident in device memory (bench `value`): stage once, then update by index.  pts = n_scans x n x 3.
    int stage_scans(const double* pts, int n_scans, int n);
    int update_staged(int index, const double* origin, const double* quat, const double odom_xyr[3], double stamp, bool* did_update);

    // sharded split-phase equivalents of update()
    int shard_begin(const double* pts, int n, const double* origin, const double* quat, const double odom_xyr[3], double stamp, bool* did_update,
                    double* local_out);
    int shard_finish(const double* all_results, bool* resampled, int32_t* idx);
    int shard_apply(const int32_t* idx, const int32_t* local_src);
    int shard_map_update();

    // Sharded operation behind update(): after shard_connect() every rank's update() runs the whole sharded step (shard_comm.h) --
    // match + map update of the local particles, ONE all-gather of the match results, the identical resampling decision on every rank,
    // NCCL send / recv of the maps of remote ancestors.
    int shard_connect(const uint8_t id[128]);
    void shard_stats(uint64_t out[2]) const { out[0] = shard_collectives_; out[1] = shard_migrated_bytes_; }
    size_t best_particle() const;                 // pf_slam2d.cpp:314-330
    double neff() const { return neff_; }
    uint32_t particles() const { return P_; }
    int local_begin() const { return lo_; }
    int local_count() const { return hi_ - lo_; }
    const SE2& pose(int i) const { return pose_[i]; }
    void weights(int i, double w[3]) const { w[0] = weight_[i]; w[1] = nweight_[i]; w[2] = wsum_[i]; }
    std::vector<SE2> trajectory(int particle) const;
    const std::vector<int32_t>& last_resample() const { return last_idx_; }
    // {number of resamplings so far, FNV-1a hash over (scan number, indices) of every one of them}: the resampling history in 16 bytes
    void resample_digest(uint64_t out[2]) const { out[0] = resample_count_; out[1] = resample_hash_; }
    // PFSlam2D::Summary buckets (include/lama/pf_slam2d.h:88-129) as host wall-clock sums in ms since creation:
    // {sampling (drawFromMotion), solve (enqueue + wait for the match results), normalise, resample (decision + device copies)}
    // getMemoryUsage() / getMemoryUsage(occmem, dmmem) (src/pf_slam2d.cpp:151-176): out = {total over all particles, occmem, dmmem}; the two-argument
    // overload of the reference adds particle 0's maps P times, which is reproduced
    int memory_usage(uint64_t out[3]);
    const std::vector<double>& timestamps() const { return timestamps_; }   // getTimestamps(): the reference records the first scan's stamp (pf_slam2d.cpp:187)
    void summary_ms(double out[4]) const { out[0] = t_sample_; out[1] = t_solve_; out[2] = t_norm_; out[3] = t_resample_; }
    const Counters& last_counters() { settle_counters(); return last_; }
    const Counters& total_counters() { settle_counters(); return total_; }
    Engine* engine() { return eng_.get(); }
    const std::string& error() const { return err_; }
    bool has_first_scan() const { return has_first_; }
    // Checkpoints (format: checkpoint.h).  save() settles the pending map update and counters, then writes the whole session without
    // changing it; a sharded handle is refused (LAMA_ERR_STATE).  load() checks the whole file before it touches CUDA (LAMA_ERR_ARG with
    // the reason in `err`), then restores on dev.device / dev.stream with dev.timing; dev.dir_dim / pool_slots / max_beams must be 0 or
    // the file's.  Kernel times, traffic counters and staged scans start empty on the loaded handle.
    int save(const std::string& path, CheckpointStats* st = nullptr);
    static PFSlam2D* load(const std::string& path, const DeviceOptions& dev, std::string& err, int* code, CheckpointStats* st = nullptr);
    bool maps_enqueued_ = false;   // sharded ranks: this scan's map update was enqueued together with its match
    int settle_counters();
    int pipelined_begin(const double* pts, int n, const double* origin, const double* quat, bool moved, bool* did_update, double* local_out);
    int update_pipelined(const double* pts, int n, const double* origin, const double* quat, const double odom_xyr[3], bool* did_update);
    void collect_map_stats(Counters& c);

private:
    PFSlam2D() = default;
    PFOptions opt_;
    std::unique_ptr<Engine> eng_;
    std::vector<double> timestamps_;
    std::mt19937 gen_;  // stands in for the reference's process-global generator (src/random.cpp:38-39)
    uint32_t P_ = 0;
    int lo_ = 0, hi_ = 0;
    std::vector<SE2> pose_;
    std::vector<double> weight_, nweight_, wsum_;
    struct Node { SE2 pose; int parent; };
    std::vector<Node> nodes_;       // ancestor-linked pose histories (Particle::poses, pf_slam2d.h:79)
    std::vector<int> node_of_;
    SE2 prior_{1, 0, 0, 0}, odom_{1, 0, 0, 0};
    bool has_first_ = false;
    double acc_trans_ = 0, acc_rot_ = 0, neff_ = 0;
    std::vector<int32_t> last_idx_;
    uint64_t resample_count_ = 0, resample_hash_ = 1469598103934665603ull, scans_seen_ = 0;
    double t_sample_ = 0, t_solve_ = 0, t_norm_ = 0, t_resample_ = 0;
    void note_resample(const std::vector<int32_t>& idx);
    Counters last_, total_;
    uint64_t detached_seen_ = 0;
    std::string err_;
    bool pending_maps_ = false, counters_pending_ = false;
    struct ShardComm* comm_ = nullptr;
    double* d_send_ = nullptr;      // device: local payload (per x kShardFields + 1 digest)
    double* d_recv_ = nullptr;      // device: gathered payloads
    double* h_recv_ = nullptr;      // pinned host copy
    int64_t* d_tab_ = nullptr;      // device: blob sizes of the particles this rank serves / of all particles
    int64_t* h_tab_ = nullptr;      // pinned
    double digest_ = 0.0;           // of the previous scan's resampling decision, compared across ranks one scan later
    uint64_t shard_collectives_ = 0, shard_migrated_bytes_ = 0;
    int update_sharded(const double* pts, int n, const double* origin, const double* quat, const double odom_xyr[3], bool* did_update);
    int migrate_and_apply(const std::vector<int32_t>& idx);
    std::vector<double> staged_host_;  // kept until the engine exists
    int staged_scans_ = 0, staged_beams_ = 0, staged_index_ = -1;
    int ensure_engine(int n);

    double rng_normal(double sigma);
    double rng_uniform();
    void draw_from_motion(const SE2& delta, SE2& p);     // :365-391
    bool predict_and_gate(const double odom_xyr[3]);      // :231-249
    int match_local(double* local_out);                   // :254-266 + scanMatch :416-437
    void absorb_results(const double* all_results);       // pose/weight bookkeeping of scanMatch
    void normalize();                                      // :511-535
    bool compute_resample(std::vector<int32_t>& idx);      // :537-553
    void apply_resample_host(const std::vector<int32_t>& idx);  // :555-573
    int first_scan(const double odom_xyr[3]);
    int fail(const std::string& m, int code) { err_ = m; return code; }
    int engine_fail(int code) { err_ = eng_->last_error(); return code; }
    void finish_counters();
};

// ---- Slam2D -----------------------------------------------------------------------------------------
struct SlamOptions {  // include/lama/slam2d.h:91-125
    double trans_thresh = 0.5, rot_thresh = 0.5, l2_max = 0.5, truncated_ray = 0.0, truncated_range = 0.0, resolution = 0.05;
    uint32_t patch_size = 32, max_iter = 100;
    int strategy = 0;
    int occupancy = 0;  // 0 = FrequencyOccupancyMap (the reference's Slam2D), 1 = ProbabilisticOccupancyMap (log-odds)
    bool transient_map = false;    // Slam2D::Options::transient_map (slam2d.h:122, slam2d.cpp:323-379)
    bool lidar_odometry = false;   // run as lama::LidarOdometry2D (src/lidar_odometry_2d.cpp:42-181): no odometry input, log-odds map,
                                   // l2_max 1.0, 1 m rays, map updated every 0.1 m / 0.5 rad, transient map always on
    DeviceOptions dev;
};

// the options and host state of a Slam2D checkpoint (every section of a kind-2 / kind-3 file but the engine), as read and checked
struct SlamSaved {
    SlamOptions opt;
    SE2 pose{1, 0, 0, 0}, odom{1, 0, 0, 0}, map_update_pose{1, 0, 0, 0};
    bool has_first = false, engine_ready = false;
    uint32_t processed = 0;
    uint64_t removed = 0, map_updates = 0;
    Counters last, total;
};

class Slam2D {
public:
    static Slam2D* create(const SlamOptions& o, std::string& err);
    void set_pose(double x, double y, double r) { pose_ = se2_from_xyr(x, y, r); }
    int update(const double* pts, int n, const double* origin, const double* quat, const double odom_xyr[3], double stamp, bool* did_update);
    const SE2& pose() const { return pose_; }
    uint32_t processed_cells() const { return processed_; }
    uint64_t removed_patches() const { return removed_; }
    uint64_t map_updates() const { return map_updates_; }
    const Counters& last_counters() const { return last_; }
    const Counters& total_counters() const { return total_; }
    Engine* engine() { return eng_.get(); }
    const DeviceOptions& device_options() const { return opt_.dev; }
    const std::string& error() const { return err_; }
    bool lidar_odometry() const { return opt_.lidar_odometry; }
    // checkpoints, as PFSlam2D::save / load; a handle saved before its first scan has no engine section
    int save(const std::string& path, CheckpointStats* st = nullptr);
    static Slam2D* load(const std::string& path, const DeviceOptions& dev, std::string& err, int* code, CheckpointStats* st = nullptr);
    // The options and state sections, shared by Slam2D files and the inner Slam2D of a GraphSlam2D file.  ckpt_get reads and checks them
    // (lidar_odometry must match the file kind); ckpt_restore builds the handle on dev.device / dev.stream with dev.timing and, when
    // `img` is given, restores its engine (*code = LAMA_ERR_CUDA when that fails).
    void ckpt_put(CkptWriter& w) const;
    static void ckpt_get(CkptReader& r, bool lidar_odometry, SlamSaved& s);
    static Slam2D* ckpt_restore(const SlamSaved& s, const EngineImage* img, const DeviceOptions& dev, std::string& err, int* code, CheckpointTimes* t);

private:
    SlamOptions opt_;
    std::unique_ptr<Engine> eng_;
    SE2 pose_{1, 0, 0, 0}, odom_{1, 0, 0, 0};
    SE2 map_update_pose_{1, 0, 0, 0};   // LidarOdometry2D::map_update_odom
    bool has_first_ = false, engine_ready_ = false;
    uint32_t processed_ = 0;
    uint64_t removed_ = 0, map_updates_ = 0;
    Counters last_, total_;
    std::string err_;
    int update_maps(const double* pts, int n);
    int update_lidar_odometry(const double* pts, int n, const double* origin, const double* quat, bool* did_update);
};

// ---- device DynamicDistanceMap + Loc2D -------------------------------------------------------------------
class DistanceMapDev {
public:
    // event_cap: addObstacle / removeObstacle calls one update() applies in a single brushfire (0 = the engine's default)
    static DistanceMapDev* create(double resolution, uint32_t patch_size, double l2_max, double cx, double cy, const DeviceOptions& dev,
                                  std::string& err, int event_cap = 0);
    int add(const uint32_t* cells_xy, int n, bool is_add);
    int update(uint32_t* processed);
    Engine* engine() { return eng_.get(); }
    const std::string& error() const { return err_; }
    int flush_if_pending();

private:
    std::unique_ptr<Engine> eng_;
    std::vector<uint32_t> pend_cells_;
    std::vector<uint8_t> pend_kind_;
    std::string err_;
};

// ---- device FrequencyOccupancyMap that keeps its own known plane: GraphSlam2D's global map ---------------------------------------------
class OccupancyMapDev {
public:
    // one-particle engine; dev.pool_slots 0 = dir_dim^2 slots, so a full window cannot run out of patches
    static OccupancyMapDev* create(double resolution, uint32_t patch_size, double cx, double cy, const DeviceOptions& dev, std::string& err);
    static OccupancyMapDev* adopt(Engine* e);   // a map around a restored engine (one particle, frequency, known plane); takes ownership
    // GraphSlam2D::generateOccupancyMap's loop body (graph_slam2d.cpp:136-160) for any posed scans (Engine::render_scans)
    int insert_scans(const double* pts, const int64_t* offsets, int n_scans, const double* origins, const double* quats, const SE2* states, bool full,
                     uint64_t* cells);
    int prune();   // FrequencyOccupancyMap::prune (frequency_occupancy_map.cpp:149-158)
    Engine* engine() { return eng_.get(); }
    const std::string& error() const { return err_; }

private:
    std::unique_ptr<Engine> eng_;
    std::string err_;
};

// ---- GraphSlam2D's loop-closure front end (src/graph_slam2d.cpp:283-355) on a device distance map -------------------------------------
// findLoopClosureCandidates (:283-313): the key poses within `radius` of `query` among the first n_keys - ignore_n (the tail of the chain is
// skipped), nearest first (nanoflann's sorted radius search), at most max_candidates.
std::vector<int> find_loop_closure_candidates(const double* key_xy, int n_keys, int ignore_n, const double query[2], double radius, int max_candidates);
// correlateCandidateScan (:315-355): the candidate's cloud matched against the map of `particle` from its own pose and from the reference
// position, one GN iteration each (Huber 0.15), the better one refined to convergence; between = matched - ref_pose, returns the
// nearest-cell RMSE (MatchSurface2D::error).
int correlate_candidate_scan(Engine* e, int particle, const double* pts, int n, const double* origin, const double* quat, const SE2& ref_pose, const SE2& cand_pose,
                             SE2* between, double* rmse);
// coarseSearchAndCorrelateCandidateScan (:357-392): first against a coarse (0.25 m, 2.5 m reach) distance map of the reference cloud alone, then
// against the map of `particle`.
int coarse_correlate_candidate_scan(Engine* e, int particle, const DeviceOptions& dev, const double* ref_pts, int ref_n, const double* ref_origin, const double* ref_quat,
                                    const double* pts, int n, const double* origin, const double* quat, const SE2& ref_pose, const SE2& cand_pose, SE2* between,
                                    double* rmse, std::string& err);

// ---- GraphSlam2D (include/lama/graph_slam2d.h:51-173, src/graph_slam2d.cpp:104-430) ----------------------------------------------------------
struct GraphOptions {  // GraphSlam2D::Options, graph_slam2d.h:59-87
    SlamOptions slam;
    double key_pose_distance = 1.0, key_pose_angular_distance = 0.5 * M_PI;
    int key_pose_head_delay = 5;
    double loop_search_max_distance = 10.0, loop_search_min_distance = 2.0;
    int loop_max_candidates = 5;
    double loop_closure_scan_rmse = 0.05;
    int loop_closure_max_candidates = 10;   // declared but read nowhere in the reference; accepted and ignored
    int ignore_n_chain_poses = 20;
};

class GraphSlam2D {
public:
    struct KeyPose {   // GraphSlam2D::KeyPose (graph_slam2d.h:97-104); `odom` is read nowhere in the reference and is not kept
        int id;
        SE2 pose, original;               // corrected (optimised) and as the inner Slam2D estimated it
        std::vector<double> pts;          // host copy of the cloud, n x 3
        double origin[3], quat[4];
        double stamp;
    };
    struct Stats {
        uint64_t loop_factors = 0, optimizations = 0, optimizations_ok = 0;
        PgoReport last;                   // of the latest optimisation
    };

    static GraphSlam2D* create(const GraphOptions& o, std::string& err);
    void init(double x, double y, double r) { slam_->set_pose(x, y, r); }   // Init (:118-121)
    // bool update(surface, odometry, timestamp) (:188-282); returns a LAMA_* status
    int update(const double* pts, int n, const double* origin, const double* quat, const double odom_xyr[3], double stamp, bool* did_update);
    SE2 pose() const { return se2_mul(correction_, slam_->pose()); }        // getPose (:127-129)
    Slam2D* slam() { return slam_.get(); }
    const std::vector<KeyPose>& key_poses() const { return keys_; }
    const std::vector<std::pair<int, int>>& links() const { return links_; }
    const std::vector<int>& last_candidates() const { return last_candidates_; }   // of the latest loop search (empty when there was none)
    const Stats& stats() const { return stats_; }
    const std::string& error() const { return err_; }
    // generateOccupancyMap (:131-164): a new map at (full ? resolution : 0.1) when mapping_keyid is 0, the key scans from mapping_keyid on
    // cast at their corrected poses, prune, mapping_keyid = number of keys.  The map is owned here and replaced on the next recreation.
    int generate_occupancy_map(bool full, OccupancyMapDev** out);
    // generateCoarseDistanceMap (:166-186): a new 0.1 m distance map (reach 5 m) with an obstacle at every occupied cell of the inner
    // Slam2D, visited in ascending directory index, then cell index; *processed = its update() return value
    int generate_coarse_distance_map(DistanceMapDev** out, uint32_t* processed);
    OccupancyMapDev* occupancy_map() { return occ_.get(); }
    DistanceMapDev* coarse_distance_map() { return coarse_dm_.get(); }
    // Checkpoints (format: checkpoint.h, kind 4), as PFSlam2D::save / load: the graph options, the inner Slam2D, the key poses with
    // their clouds, the pose graph and loop bookkeeping, the inner engine and -- when the next generate_occupancy_map would reuse it --
    // the global map.  The coarse distance map is rebuilt by every generate_coarse_distance_map and is not saved.
    int save(const std::string& path, CheckpointStats* st = nullptr);
    static GraphSlam2D* load(const std::string& path, const DeviceOptions& dev, std::string& err, int* code, CheckpointStats* st = nullptr);

private:
    GraphOptions opt_;
    std::unique_ptr<Slam2D> slam_;
    size_t mapping_keyid_ = 0;                      // graph_slam2d.h: the first key not yet cast into occ_
    std::unique_ptr<OccupancyMapDev> occ_;
    std::unique_ptr<DistanceMapDev> coarse_dm_;
    std::vector<KeyPose> keys_;
    std::vector<std::pair<int, int>> links_;
    std::vector<PgoPrior> priors_;            // the persistent graph (graph_slam2d.cpp:110): the prior on key 0,
    std::vector<PgoBetween> factors_;         // then chain and loop factors in graph->add order
    std::vector<PgoBetween> queue_;           // factor_queue: loop factors not yet in the graph
    std::vector<int> last_candidates_;
    SE2 correction_{1, 0, 0, 0};
    double accdist_ = 0.0;
    // the function-local statics of update() (:197, :200, :244) kept per instance: the reference shares them across every
    // GraphSlam2D of a process; for a single instance the behaviour is the same
    SE2 prev_ = se2_from_xyr(1e10, 1e10, 0.0);
    double factordist_ = 0.0;
    Stats stats_;
    std::string err_;
    GraphSlam2D() = default;
    int optimize_pose_graph();                 // optimizePoseGraph (:394-430)
};

// SimpleOccupancyMap (src/sdm/simple_occupancy_map.cpp:36-149): Loc2D's static tri-state map.  It is only consulted by
// the host-side rejection sampling of globalLocalization, so it lives on the host.
class SimpleOccupancyHost {
public:
    explicit SimpleOccupancyHost(double resolution) : resolution_(resolution), scale_(1.0 / resolution) {}
    double resolution() const { return resolution_; }
    void set(uint32_t x, uint32_t y, int state);   // -1 setFree, 0 setUnknown, 1 setOccupied
    bool is_free_world(double wx, double wy) const;
    bool bounds_world(double mn[2], double mx[2]) const;  // Map::bounds, patch granular (map.cpp:119-138)
private:
    double resolution_, scale_;
    std::unordered_map<uint64_t, std::vector<int8_t>> patches_;
};

struct LocOptions {  // src/loc2d.cpp:46-58
    double trans_thresh = 0.5, rot_thresh = 0.5, l2_max = 1.0, resolution = 0.05;
    uint32_t patch_size = 32, max_iter = 100;
    int strategy = 0;
    uint32_t gloc_particles = 3000, gloc_iters = 10;
    double gloc_thresh = 0.15, cov_blend = 0.0;
    double center_x = 0, center_y = 0;
    DeviceOptions dev;
};

class Loc2D {
public:
    static Loc2D* create(const LocOptions& o, std::string& err);
    DistanceMapDev* distance_map() { return dm_.get(); }
    SimpleOccupancyHost* occupancy_map() { return occ_.get(); }
    void set_seed(uint32_t seed) { gen_.seed(seed); }                 // random::setSeed
    void trigger_global_localization() { do_gloc_ = true; }          // loc2d.cpp:194-197
    bool global_localization_active() const { return do_gloc_; }
    void set_pose(double x, double y, double r)
    {
        pose_      = se2_from_xyr(x, y, r);
        has_first_ = false;
    }
    int update(const double* pts, int n, const double* origin, const double* quat, const double odom_xyr[3], double stamp, bool force, bool* did_update);
    const SE2& pose() const { return pose_; }
    const double* cov() const { return cov_; }
    double rmse() const { return rmse_; }
    uint32_t iterations() const { return iters_; }
    uint32_t evals() const { return evals_; }
    const std::string& error() const { return err_; }

private:
    LocOptions opt_;
    std::unique_ptr<DistanceMapDev> dm_;
    SE2 pose_{1, 0, 0, 0}, odom_{1, 0, 0, 0};
    bool has_first_ = false;
    double cov_[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    double rmse_ = 0;
    uint32_t iters_ = 0, evals_ = 0;
    std::string err_;
    std::unique_ptr<SimpleOccupancyHost> occ_;
    std::mt19937 gen_{std::random_device{}()};   // the reference's global generator is seeded from random_device (random.cpp:38-39)
    bool do_gloc_ = false;
    uint32_t gloc_cur_iter_ = 0;
    double cov_blend_ = 0.0;
    std::vector<double> sampling_steps_;         // 161 (x, y) offsets, loc2d.cpp:93-107
    int global_localization(int n);               // loc2d.cpp:249-286
    int add_sampling_covariance(int n);           // loc2d.cpp:199-247
};

// shared helpers
SolverOptions make_solver(int strategy, uint32_t max_iter);
void covariance_from_sums(const double sums[kNumSums], size_t rows, double cov[9]);  // Solver::calculateCovariance, solver.cpp:133-150
void unpack_distance_words(const uint32_t* words, const uint8_t* occ_known, size_t n, uint16_t* sqdist, uint8_t* valid, uint8_t* known, int16_t* ox,
                           int16_t* oy, uint8_t* queued);

}  // namespace lama_b200
