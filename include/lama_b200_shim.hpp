// lama_b200_shim.hpp -- header-only C++ shim that re-creates the reference's front-end classes on top of the C-ABI.
//
// A maintainer of iris-ua/iris_lama would add this file next to include/lama/pf_slam2d.h and let
// lama::PFSlam2D / Slam2D / Loc2D forward to it (see INTEGRATION.md).  It is templated on the caller's
// point-cloud and pose types so that it compiles without Eigen: any cloud with `.points` (elements indexable
// [0..2]), `.sensor_origin_` (indexable [0..2]) and `.sensor_orientation_` (with x(), y(), z(), w()) works,
// i.e. lama::PointCloudXYZ (include/lama/types.h:111-120); any pose with x(), y(), rotation() works, i.e.
// lama::Pose2D (include/lama/pose2d.h:42-78).
#pragma once

#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "lama_b200.h"

namespace lama_b200_shim {

inline void check(int rc)
{
    if (rc != LAMA_OK) throw std::runtime_error(std::string("lama_b200: ") + lama_last_error());
}

template <typename Cloud>
struct FlatCloud {
    std::vector<double> pts;
    double origin[3], quat[4];
    explicit FlatCloud(const Cloud& c)
    {
        pts.reserve(c.points.size() * 3);
        for (const auto& p : c.points) { pts.push_back(p[0]); pts.push_back(p[1]); pts.push_back(p[2]); }
        for (int i = 0; i < 3; ++i) origin[i] = c.sensor_origin_[i];
        quat[0] = c.sensor_orientation_.x(); quat[1] = c.sensor_orientation_.y();
        quat[2] = c.sensor_orientation_.z(); quat[3] = c.sensor_orientation_.w();
    }
};

// lama::PFSlam2D (include/lama/pf_slam2d.h:187-232)
// the maps' working window (lama_pf_get_window / lama_slam_get_window): base in patch coordinates, dir_dim, shifts so far, entries
// parked outside the window now, entries restored so far
struct MapWindow {
    int32_t base[2] = {0, 0};
    int32_t dim = 0;
    uint64_t shifts = 0, parked = 0, restored = 0;
};
inline MapWindow map_window(int rc, const int32_t base[2], int32_t dim, const uint64_t c[3])
{
    check(rc);
    MapWindow w;
    w.base[0] = base[0]; w.base[1] = base[1]; w.dim = dim;
    w.shifts = c[0]; w.parked = c[1]; w.restored = c[2];
    return w;
}

// a device FrequencyOccupancyMap (lama_om, stand-alone or the global map GraphSlam2D::generateOccupancyMap returns): following on or off
// (lama_om_set_follow; a GraphSlam2D's map always follows), its working window and its pool {slots, slots in use}
inline void occupancyMapSetFollow(lama_om* m, bool on) { check(lama_om_set_follow(m, on ? 1 : 0)); }
inline MapWindow occupancyMapWindow(lama_om* m)
{
    int32_t b[2], d = 0;
    uint64_t c[3];
    return map_window(lama_om_get_window(m, b, &d, c), b, d, c);
}
inline void occupancyMapPool(lama_om* m, uint64_t out[2]) { check(lama_om_get_pool(m, out)); }

// a device DynamicDistanceMap (lama_dm, stand-alone or a Loc2D's distance_map()): following on or off (lama_dm_set_follow; a Loc2D
// follows exactly when its distance map does), its working window and its pool {slots, slots in use}
inline void distanceMapSetFollow(lama_dm* m, bool on) { check(lama_dm_set_follow(m, on ? 1 : 0)); }
inline MapWindow distanceMapWindow(lama_dm* m)
{
    int32_t b[2], d = 0;
    uint64_t c[3];
    return map_window(lama_dm_get_window(m, b, &d, c), b, d, c);
}
inline void distanceMapPool(lama_dm* m, uint64_t out[2]) { check(lama_dm_get_pool(m, out)); }

class PFSlam2D {
public:
    using Options = lama_pf_options;
    static Options defaults(uint32_t particles)
    {
        Options o;
        check(lama_pf_options_default(&o));
        o.particles = particles;
        return o;
    }
    explicit PFSlam2D(const Options& o) { check(lama_pf_create(&o, &h_)); }
    ~PFSlam2D() { lama_pf_destroy(h_); }
    PFSlam2D(const PFSlam2D&) = delete;
    PFSlam2D& operator=(const PFSlam2D&) = delete;

    template <typename Pose>
    void setPrior(const Pose& prior)  // pf_slam2d.cpp:146-149
    {
        const double xyr[3] = {prior.x(), prior.y(), prior.rotation()};
        check(lama_pf_set_prior(h_, xyr));
    }
    // bool update(const PointCloudXYZ::Ptr& surface, const Pose2D& odometry, double timestamp)  pf_slam2d.h:199
    template <typename CloudPtr, typename Pose>
    bool update(const CloudPtr& surface, const Pose& odometry, double timestamp)
    {
        FlatCloud<typename std::remove_reference<decltype(*surface)>::type> f(*surface);
        const double odom[3] = {odometry.x(), odometry.y(), odometry.rotation()};
        int did = 0;
        check(lama_pf_update(h_, f.pts.data(), (int)(f.pts.size() / 3), f.origin, f.quat, odom, timestamp, &did));
        return did != 0;
    }
    void getPose(double xyr[3]) const { check(lama_pf_get_pose(h_, xyr)); }       // pf_slam2d.cpp:332-336
    size_t getBestParticleIdx() const { int i = 0; check(lama_pf_get_best_particle(h_, &i)); return (size_t)i; }
    double getNeff() const { double v = 0; check(lama_pf_get_neff(h_, &v)); return v; }
    // Map::write of a particle's occupancy (kind 0) / distance (kind 1) map: a reference .sdm file (map.cpp:490-529)
    void writeMap(int particle, int kind, const std::string& path) const { check(lama_pf_write_map(h_, particle, kind, path.c_str())); }
    // the grey image PFSlam2D::saveOccImage hands to sdm::export_to_png (pf_slam2d.cpp:338-342, export.cpp:46-73), row-major
    std::vector<uint8_t> occImage(int& width, int& height) const
    {
        int dims[2] = {0, 0};
        const int best = (int)getBestParticleIdx();
        check(lama_pf_export_image(h_, best, 0, nullptr, 0, dims));
        std::vector<uint8_t> img((size_t)dims[0] * dims[1]);
        if (!img.empty()) check(lama_pf_export_image(h_, best, 0, img.data(), img.size(), dims));
        width = dims[0]; height = dims[1];
        return img;
    }
    lama_pf* handle() const { return h_; }
    // checkpoints (no counterpart in the reference): the whole session to a file, and a filter that continues it bit for bit
    void saveState(const std::string& path) const { check(lama_pf_save_state(h_, path.c_str())); }
    static std::unique_ptr<PFSlam2D> loadState(const std::string& path, int device = 0)
    {
        lama_device_options dev = {device, 0, 0, 0, 0, 0};
        lama_pf* h = nullptr;
        check(lama_pf_load_state(path.c_str(), &dev, &h));
        return std::unique_ptr<PFSlam2D>(new PFSlam2D(h));
    }
    // sharded sessions: each rank saves its shard; any complete set (or one saveState file) loads as rank shard_rank of shard_count
    void saveShardState(const std::string& path) const { check(lama_pf_save_shard_state(h_, path.c_str())); }
    static std::unique_ptr<PFSlam2D> loadStateSharded(const std::vector<std::string>& paths, uint32_t shard_rank, uint32_t shard_count, int device = 0)
    {
        lama_device_options dev = {device, 0, 0, 0, 0, 0};
        std::vector<const char*> p;
        for (const std::string& s : paths) p.push_back(s.c_str());
        lama_pf* h = nullptr;
        check(lama_pf_load_state_sharded(p.data(), (int)p.size(), shard_rank, shard_count, &dev, &h));
        return std::unique_ptr<PFSlam2D>(new PFSlam2D(h));
    }

    MapWindow window() const
    {
        int32_t b[2], d = 0;
        uint64_t c[3];
        return map_window(lama_pf_get_window(h_, b, &d, c), b, d, c);
    }

private:
    explicit PFSlam2D(lama_pf* h) : h_(h) {}
    lama_pf* h_ = nullptr;
};

// lama::Slam2D (include/lama/slam2d.h:128-161)
class Slam2D {
public:
    using Options = lama_slam_options;
    static Options defaults() { Options o; check(lama_slam_options_default(&o)); return o; }
    explicit Slam2D(const Options& o) { check(lama_slam_create(&o, &h_)); }
    ~Slam2D() { lama_slam_destroy(h_); }
    Slam2D(const Slam2D&) = delete;
    Slam2D& operator=(const Slam2D&) = delete;
    template <typename Pose>
    void setPose(const Pose& p) { const double xyr[3] = {p.x(), p.y(), p.rotation()}; check(lama_slam_set_pose(h_, xyr)); }
    template <typename CloudPtr, typename Pose>
    bool update(const CloudPtr& surface, const Pose& odometry, double timestamp)  // slam2d.h:134
    {
        FlatCloud<typename std::remove_reference<decltype(*surface)>::type> f(*surface);
        const double odom[3] = {odometry.x(), odometry.y(), odometry.rotation()};
        int did = 0;
        check(lama_slam_update(h_, f.pts.data(), (int)(f.pts.size() / 3), f.origin, f.quat, odom, timestamp, &did));
        return did != 0;
    }
    void getPose(double xyr[3]) const { check(lama_slam_get_pose(h_, xyr)); }
    uint32_t getNumberOfProcessedCells() const { uint32_t n = 0; check(lama_slam_get_processed_cells(h_, &n)); return n; }
    void writeMap(int kind, const std::string& path) const { check(lama_slam_write_map(h_, kind, path.c_str())); }
    lama_slam* handle() const { return h_; }
    MapWindow window() const
    {
        int32_t b[2], d = 0;
        uint64_t c[3];
        return map_window(lama_slam_get_window(h_, b, &d, c), b, d, c);
    }
    // checkpoints (no counterpart in the reference), as PFSlam2D::saveState / loadState
    void saveState(const std::string& path) const { check(lama_slam_save_state(h_, path.c_str())); }
    static std::unique_ptr<Slam2D> loadState(const std::string& path, int device = 0)
    {
        lama_device_options dev = {device, 0, 0, 0, 0, 0};
        lama_slam* h = nullptr;
        check(lama_slam_load_state(path.c_str(), &dev, &h));
        return std::unique_ptr<Slam2D>(new Slam2D(h));
    }

protected:
    explicit Slam2D(lama_slam* h) : h_(h) {}
    lama_slam* h_ = nullptr;
};

// lama::GraphSlam2D (include/lama/graph_slam2d.h:51-173): key-pose graph SLAM over a transient-map Slam2D
class GraphSlam2D {
public:
    using Options = lama_graph_options;
    static Options defaults() { Options o; check(lama_graph_options_default(&o)); return o; }
    explicit GraphSlam2D(const Options& o = defaults()) { check(lama_graph_create(&o, &h_)); }
    ~GraphSlam2D() { lama_graph_destroy(h_); }
    GraphSlam2D(const GraphSlam2D&) = delete;
    GraphSlam2D& operator=(const GraphSlam2D&) = delete;
    template <typename Pose>
    void Init(const Pose& prior) { const double xyr[3] = {prior.x(), prior.y(), prior.rotation()}; check(lama_graph_set_pose(h_, xyr)); }   // :118-121
    template <typename CloudPtr, typename Pose>
    bool update(const CloudPtr& surface, const Pose& odometry, double timestamp)  // graph_slam2d.h:150
    {
        FlatCloud<typename std::remove_reference<decltype(*surface)>::type> f(*surface);
        const double odom[3] = {odometry.x(), odometry.y(), odometry.rotation()};
        int did = 0;
        check(lama_graph_update(h_, f.pts.data(), (int)(f.pts.size() / 3), f.origin, f.quat, odom, timestamp, &did));
        return did != 0;
    }
    void getPose(double xyr[3]) const { check(lama_graph_get_pose(h_, xyr)); }   // :127-129
    // the inner Slam2D (the public member `slam`), borrowed: valid while this object lives
    lama_slam* slam() const { lama_slam* s = nullptr; check(lama_graph_slam(h_, &s)); return s; }
    // generateOccupancyMap (:131-164) / generateCoarseDistanceMap (:166-186): BORROWED maps, owned by this object and replaced in
    // place when it recreates them (the reference returns a fresh shared_ptr instead)
    lama_om* generateOccupancyMap(bool full = false) { lama_om* m = nullptr; check(lama_graph_generate_occupancy_map(h_, full ? 1 : 0, &m)); return m; }
    lama_dm* generateCoarseDistanceMap() { lama_dm* d = nullptr; check(lama_graph_generate_coarse_distance_map(h_, &d, nullptr)); return d; }
    lama_graph* handle() const { return h_; }
    // checkpoints (no counterpart in the reference), as PFSlam2D::saveState / loadState
    void saveState(const std::string& path) const { check(lama_graph_save_state(h_, path.c_str())); }
    static std::unique_ptr<GraphSlam2D> loadState(const std::string& path, int device = 0)
    {
        lama_device_options dev = {device, 0, 0, 0, 0, 0};
        lama_graph* h = nullptr;
        check(lama_graph_load_state(path.c_str(), &dev, &h));
        return std::unique_ptr<GraphSlam2D>(new GraphSlam2D(h));
    }

private:
    explicit GraphSlam2D(lama_graph* h) : h_(h) {}
    lama_graph* h_ = nullptr;
};

// lama::LidarOdometry2D (include/lama/lidar_odometry_2d.h:45-75): the Slam2D handle in its lidar-odometry mode
class LidarOdometry2D {
public:
    struct Options {
        double resolution;
        uint32_t max_iter;
        Options() : resolution(0.05), max_iter(100) {}   // lidar_odometry_2d.h:62-68
    };
    explicit LidarOdometry2D(const Options& o = Options())
    {
        lama_slam_options s;
        check(lama_slam_options_default(&s));
        s.lidar_odometry = 1; s.resolution = o.resolution; s.max_iter = o.max_iter;
        check(lama_slam_create(&s, &h_));
    }
    ~LidarOdometry2D() { lama_slam_destroy(h_); }
    LidarOdometry2D(const LidarOdometry2D&) = delete;
    LidarOdometry2D& operator=(const LidarOdometry2D&) = delete;
    template <typename CloudPtr>
    bool update(const CloudPtr& surface, double timestamp)  // lidar_odometry_2d.h:73
    {
        FlatCloud<typename std::remove_reference<decltype(*surface)>::type> f(*surface);
        int did = 0;
        check(lama_slam_update(h_, f.pts.data(), (int)(f.pts.size() / 3), f.origin, f.quat, nullptr, timestamp, &did));
        return did != 0;
    }
    void getOdom(double xyr[3]) const { check(lama_slam_get_pose(h_, xyr)); }   // the public member `odom`
    MapWindow window() const
    {
        int32_t b[2], d = 0;
        uint64_t c[3];
        return map_window(lama_slam_get_window(h_, b, &d, c), b, d, c);
    }

private:
    lama_slam* h_ = nullptr;
};

// lama::Loc2D (include/lama/loc2d.h:103-130); the caller fills distance_map() through lama_dm_add_obstacles + lama_dm_update
class Loc2D {
public:
    using Options = lama_loc_options;
    static Options defaults() { Options o; check(lama_loc_options_default(&o)); return o; }
    void Init(const Options& o) { check(lama_loc_create(&o, &h_)); }
    ~Loc2D() { lama_loc_destroy(h_); }
    lama_dm* distance_map() { lama_dm* d = nullptr; check(lama_loc_distance_map(h_, &d)); return d; }
    template <typename Pose>
    void setPose(const Pose& p) { const double xyr[3] = {p.x(), p.y(), p.rotation()}; check(lama_loc_set_pose(h_, xyr)); }
    template <typename CloudPtr, typename Pose>
    bool update(const CloudPtr& surface, const Pose& odometry, double timestamp, bool force_update = false)  // loc2d.h:113
    {
        FlatCloud<typename std::remove_reference<decltype(*surface)>::type> f(*surface);
        const double odom[3] = {odometry.x(), odometry.y(), odometry.rotation()};
        int did = 0;
        check(lama_loc_update(h_, f.pts.data(), (int)(f.pts.size() / 3), f.origin, f.quat, odom, timestamp, force_update ? 1 : 0, &did));
        return did != 0;
    }
    void getPose(double xyr[3]) const { check(lama_loc_get_pose(h_, xyr)); }
    void getCovar(double cov[9]) const { check(lama_loc_get_covar(h_, cov)); }
    double getRMSE() const { double v = 0; check(lama_loc_get_rmse(h_, &v)); return v; }
    void triggerGlobalLocalization() { check(lama_loc_trigger_global_localization(h_)); }   // loc2d.cpp:194-197
    void readOccupancyMap(const std::string& path) { check(lama_loc_occupancy_read(h_, path.c_str())); }    // occupancy_map->read(path)
    void readDistanceMap(const std::string& path) { check(lama_dm_read(distance_map(), path.c_str())); }    // distance_map->read(path)
    // following on or off, through the distance map (lama_dm_set_follow); turn it on before readDistanceMap for a map larger than the window
    void setFollow(bool on) { distanceMapSetFollow(distance_map(), on); }
    MapWindow window() { return distanceMapWindow(distance_map()); }

private:
    lama_loc* h_ = nullptr;
};

// lama::TruncatedSignedDistanceMap (include/lama/sdm/truncated_signed_distance_map.h) on the device; toMesh gives the vertices
// (3 per triangle, index[i] = i), writePly is sdm::export_to_ply
class TruncatedSignedDistanceMap {
public:
    explicit TruncatedSignedDistanceMap(double resolution, uint32_t patch_size = 32, bool is3d = false)
    {
        check(lama_tsdm_create(resolution, patch_size, is3d ? 1 : 0, nullptr, nullptr, nullptr, &h_));
    }
    ~TruncatedSignedDistanceMap() { lama_tsdm_destroy(h_); }
    TruncatedSignedDistanceMap(const TruncatedSignedDistanceMap&) = delete;
    TruncatedSignedDistanceMap& operator=(const TruncatedSignedDistanceMap&) = delete;
    template <typename CloudPtr>
    size_t insertPointCloud(const CloudPtr& cloud)   // truncated_signed_distance_map.cpp:141-158
    {
        FlatCloud<typename std::remove_reference<decltype(*cloud)>::type> f(*cloud);
        const int64_t offsets[2] = {0, (int64_t)(f.pts.size() / 3)};
        uint64_t n = 0;
        check(lama_tsdm_insert_point_clouds(h_, f.pts.data(), offsets, 1, f.origin, f.quat, &n));
        return (size_t)n;
    }
    double distance(const double xyz[3], double gradient[3] = nullptr) const { double d = 0; check(lama_tsdm_distance(h_, xyz, 1, &d, gradient)); return d; }
    void setMaxDistance(double d) { check(lama_tsdm_set_max_distance(h_, d)); }
    double maxDistance() const { double d = 0; check(lama_tsdm_max_distance(h_, &d)); return d; }
    std::vector<float> toMesh() const   // x, y, z per vertex
    {
        size_t n = 0;
        check(lama_tsdm_to_mesh(h_, nullptr, 0, &n));
        std::vector<float> v(n * 3);
        if (n) check(lama_tsdm_to_mesh(h_, v.data(), n, &n));
        return v;
    }
    void writePly(const std::string& path) const { check(lama_tsdm_write_ply(h_, path.c_str())); }

private:
    lama_tsdm* h_ = nullptr;
};

class DynamicDistanceMap3D;

// lama::FrequencyOccupancyMap (kind 0) / lama::ProbabilisticOccupancyMap (kind 1) with is3d = true on the device.  Cells are map
// coordinates {x, y, z}; insertPointCloud is the loop body of GraphSlam2D::generateOccupancyMap for every point of the cloud.
class OccupancyMap3D {
public:
    explicit OccupancyMap3D(double resolution, int kind = 0, uint32_t patch_size = 32)
    {
        check(lama_om3_create(resolution, patch_size, kind, nullptr, nullptr, nullptr, &h_));
    }
    ~OccupancyMap3D() { lama_om3_destroy(h_); }
    OccupancyMap3D(const OccupancyMap3D&) = delete;
    OccupancyMap3D& operator=(const OccupancyMap3D&) = delete;
    template <typename CloudPtr>
    uint64_t insertPointCloud(const CloudPtr& cloud, bool full = true)   // graph_slam2d.cpp:146-158; returns the cell updates
    {
        FlatCloud<typename std::remove_reference<decltype(*cloud)>::type> f(*cloud);
        const int64_t offsets[2] = {0, (int64_t)(f.pts.size() / 3)};
        uint64_t n = 0;
        check(lama_om3_insert_point_clouds(h_, f.pts.data(), offsets, 1, f.origin, f.quat, full ? 1 : 0, &n));
        return n;
    }
    // the map update of Slam2D::updateMaps (slam2d.cpp:271-316) for the cloud with dm kept in step; returns dm.update()'s count
    template <typename CloudPtr>
    uint32_t updateMaps(DynamicDistanceMap3D& dm, const CloudPtr& cloud, bool full = true);
    bool setFree(const uint32_t xyz[3]) { return set(xyz, LAMA_OM3_SET_FREE); }
    bool setOccupied(const uint32_t xyz[3]) { return set(xyz, LAMA_OM3_SET_OCCUPIED); }
    bool setUnknown(const uint32_t xyz[3]) { return set(xyz, LAMA_OM3_SET_UNKNOWN); }
    bool isFree(const uint32_t xyz[3]) const { return (flags(xyz) & 1) != 0; }
    bool isOccupied(const uint32_t xyz[3]) const { return (flags(xyz) & 2) != 0; }
    bool isUnknown(const uint32_t xyz[3]) const { return (flags(xyz) & 4) != 0; }
    double getProbability(const uint32_t xyz[3]) const { double p = 0; uint8_t f = 0; check(lama_om3_query(h_, xyz, 1, &p, &f)); return p; }
    void prune() { check(lama_om3_prune(h_)); }
    bool write(const std::string& path) const { check(lama_om3_write(h_, path.c_str())); return true; }
    bool read(const std::string& path) { check(lama_om3_read(h_, path.c_str())); return true; }

private:
    bool set(const uint32_t xyz[3], uint8_t op) { uint8_t c = 0; check(lama_om3_apply(h_, xyz, &op, 1, &c)); return c != 0; }
    uint8_t flags(const uint32_t xyz[3]) const { double p = 0; uint8_t f = 0; check(lama_om3_query(h_, xyz, 1, &p, &f)); return f; }
    lama_om3* h_ = nullptr;
};

// lama::DynamicDistanceMap with is3d = true on the device.  Cells are map coordinates {x, y, z}; setMaxDistance is fixed at creation
// (l2_max).  addObstacle / removeObstacle are queued and applied by update() or the next read of the map.
class DynamicDistanceMap3D {
public:
    explicit DynamicDistanceMap3D(double resolution, double l2_max = 0.5, uint32_t patch_size = 32)
    {
        check(lama_dm3_create(resolution, patch_size, l2_max, nullptr, nullptr, nullptr, &h_));
    }
    ~DynamicDistanceMap3D() { lama_dm3_destroy(h_); }
    DynamicDistanceMap3D(const DynamicDistanceMap3D&) = delete;
    DynamicDistanceMap3D& operator=(const DynamicDistanceMap3D&) = delete;
    void addObstacle(const uint32_t xyz[3]) { check(lama_dm3_add_obstacles(h_, xyz, 1)); }         // dynamic_distance_map.cpp:212-226
    void removeObstacle(const uint32_t xyz[3]) { check(lama_dm3_remove_obstacles(h_, xyz, 1)); }   // :228-242
    uint32_t update() { uint32_t n = 0; check(lama_dm3_update(h_, &n)); return n; }                // :160-197
    double distance(const double xyz[3], double gradient[3] = nullptr) const { double d = 0; check(lama_dm3_distance(h_, xyz, 1, &d, gradient)); return d; }
    double distance(const uint32_t xyz[3]) const { double d = 0; check(lama_dm3_cell_distance(h_, xyz, 1, &d)); return d; }
    double maxDistance() const { double d = 0; check(lama_dm3_max_distance(h_, &d)); return d; }
    bool write(const std::string& path) const { check(lama_dm3_write(h_, path.c_str())); return true; }
    bool read(const std::string& path) { check(lama_dm3_read(h_, path.c_str())); return true; }

private:
    friend class OccupancyMap3D;
    lama_dm3* h_ = nullptr;
};

template <typename CloudPtr>
uint32_t OccupancyMap3D::updateMaps(DynamicDistanceMap3D& dm, const CloudPtr& cloud, bool full)
{
    FlatCloud<typename std::remove_reference<decltype(*cloud)>::type> f(*cloud);
    const int64_t offsets[2] = {0, (int64_t)(f.pts.size() / 3)};
    uint32_t processed = 0;
    check(lama_om3_insert_point_clouds_dm3(h_, dm.h_, f.pts.data(), offsets, 1, f.origin, f.quat, full ? 1 : 0, nullptr, &processed, nullptr));
    return processed;
}

}  // namespace lama_b200_shim
