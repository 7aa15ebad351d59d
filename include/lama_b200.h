/* lama_b200.h -- C-ABI of the H100-native (sm_90a) LaMa hot path (liblama_b200.so).
 *
 * The reference (iris-ua/iris_lama) has no plugin / FFI layer: the particle-filter SLAM hot path sits
 * behind plain C++ classes.  Every entry point below names the reference interface it replaces
 * (paths relative to the reference tree).  Plain pointers and sizes only; every function returns an
 * int status (0 = ok, < 0 = error, see LAMA_ERR_*) and lama_last_error() gives the message.
 * Handles are not thread safe: one host thread per handle (as the reference objects).
 *
 * Conventions
 *   poses       xyr[3] = (x, y, rotation) like lama::Pose2D(x, y, rotation), include/lama/pose2d.h:45
 *   SE2 states  state[4] = (cos, sin, tx, ty): the raw Sophus SE2 of Pose2D::state, pose2d.h:76
 *   scans       pts_xyz = N x 3 doubles (PointCloudXYZ::points), sensor_origin[3], sensor_quat_xyzw[4]
 *               (PointCloudXYZ::sensor_origin_ / sensor_orientation_), include/lama/types.h:111-120
 *   map cells   absolute unsigned map coordinates as produced by Map::w2m, include/lama/sdm/map.h:125
 */
#ifndef LAMA_B200_H
#define LAMA_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LAMA_OK 0
#define LAMA_ERR_ARG (-1)
#define LAMA_ERR_CUDA (-2)
#define LAMA_ERR_NO_DEVICE (-3)
#define LAMA_ERR_WINDOW (-4)   /* the map grew outside the device directory window (raise dir_dim) */
#define LAMA_ERR_POOL (-5)     /* device patch pool exhausted (raise pool_slots) */
#define LAMA_ERR_OVERFLOW (-6) /* per-scan event log / brushfire heap overflow */
#define LAMA_ERR_STATE (-7)

/* message of the last failing call on this thread */
const char* lama_last_error(void);
/* library / build identification, e.g. "lama_b200 0.1 sm_90a" */
const char* lama_version(void);
/* number of visible CUDA devices (0 when none: every create call then fails with LAMA_ERR_NO_DEVICE) */
int lama_device_count(void);

/* device-side knobs shared by all front ends (no counterpart in the reference) */
typedef struct lama_device_options {
    int32_t device;      /* CUDA device ordinal */
    int32_t dir_dim;     /* map window = dir_dim x dir_dim patches of 32 x 32 cells, power of two, default 64 */
    int32_t pool_slots;  /* 4 KiB patches in the device pool, 0 = auto */
    int32_t max_beams;   /* largest scan accepted, default 2048 */
    int32_t timing;      /* 1: record CUDA-event times per kernel (lama_*_kernel_times) */
    uint64_t stream;     /* cudaStream_t to launch on (e.g. a torch stream), 0 = the handle creates its own */
} lama_device_options;

/* ------------------------------------------------------------------------------------------------
 * PFSlam2D -- include/lama/pf_slam2d.h:132-232, src/pf_slam2d.cpp:106-574
 * ------------------------------------------------------------------------------------------------ */
typedef struct lama_pf lama_pf;

typedef struct lama_pf_options { /* PFSlam2D::Options, pf_slam2d.h:132-185 */
    uint32_t particles;
    double srr, str, stt, srt;
    double meas_sigma, meas_sigma_gain;
    double trans_thresh, rot_thresh;
    double l2_max;
    double truncated_ray, truncated_range;
    double resolution;
    uint32_t patch_size; /* must be 32 */
    uint32_t max_iter;
    int32_t strategy;    /* 0 "gn", 1 "lm" (PFSlam2D::scanMatch always uses Gauss-Newton, pf_slam2d.cpp:423-427) */
    int32_t threads;     /* accepted for source compatibility; the particle loop runs on the GPU */
    uint32_t seed;       /* 0 = random_device, pf_slam2d.cpp:131-134 */
    /* particle sharding over GPUs (one process per GPU): this handle owns particles
       [shard_rank * particles / shard_count, (shard_rank + 1) * particles / shard_count) */
    uint32_t shard_rank, shard_count;
    lama_device_options dev;
} lama_pf_options;

/* fills the reference defaults (pf_slam2d.h:132-185); `particles` has none there and is set to 1 */
int lama_pf_options_default(lama_pf_options* o);
/* PFSlam2D::PFSlam2D(const Options&), pf_slam2d.cpp:106-138 */
int lama_pf_create(const lama_pf_options* o, lama_pf** out);
int lama_pf_destroy(lama_pf* h);
/* PFSlam2D::setPrior, pf_slam2d.cpp:146-149 */
int lama_pf_set_prior(lama_pf* h, const double xyr[3]);
/* bool PFSlam2D::update(surface, odometry, timestamp), pf_slam2d.cpp:178-312; *did_update = the bool */
int lama_pf_update(lama_pf* h, const double* pts_xyz, int n, const double sensor_origin[3], const double sensor_quat_xyzw[4],
                   const double odom_xyr[3], double timestamp, int* did_update);
/* Device-resident inputs: copy n_scans x n x 3 doubles into HBM once, then run update() on scan `index`
   without any host->device transfer of points (same semantics as lama_pf_update otherwise) */
int lama_pf_stage_scans(lama_pf* h, const double* pts_xyz, int n_scans, int n);
int lama_pf_update_staged(lama_pf* h, int index, const double sensor_origin[3], const double sensor_quat_xyzw[4], const double odom_xyr[3],
                          double timestamp, int* did_update);
/* bytes moved host->device [0] and device->host [1] by the update path since the last reset (reset != 0 also
   clears the kernel timers) */
int lama_pf_get_traffic(lama_pf* h, uint64_t bytes[2], int reset);
/* PFSlam2D::getPose (best particle), pf_slam2d.cpp:332-336 */
int lama_pf_get_pose(lama_pf* h, double xyr[3]);
int lama_pf_get_best_particle(lama_pf* h, int* idx);      /* getBestParticleIdx, pf_slam2d.cpp:314-330 */
int lama_pf_get_neff(lama_pf* h, double* neff);           /* getNeff, pf_slam2d.h:229 */
/* getParticles(): states P x 4, weights P x 3 = (weight, normalized_weight, weight_sum); either may be NULL */
int lama_pf_get_particles(lama_pf* h, double* states, double* weights);
/* Particle::poses history of one particle as xyr triples; returns the length in *count (cap = capacity) */
int lama_pf_get_trajectory(lama_pf* h, int particle, double* xyr, int cap, int* count);
/* indices drawn by the last PFSlam2D::resample (pf_slam2d.cpp:537-574); *count = 0 when the last update did not resample */
int lama_pf_get_last_resample(lama_pf* h, int32_t* idx, int* count);
/* The whole resampling history in 16 bytes: out[0] = resamplings so far (Summary::resample count, pf_slam2d.h:88-129), out[1] = FNV-1a
 * hash over (accepted-scan number, the P ancestor indices) of each of them, bytes little endian (src/pf_slam2d.cpp:537-553). */
int lama_pf_get_resample_digest(lama_pf* h, uint64_t out[2]);
/* PFSlam2D::Summary time buckets (include/lama/pf_slam2d.h:88-129, filled at src/pf_slam2d.cpp:251-311) as host wall-clock sums in ms:
 * {sampling (drawFromMotion), solve (scan matching: enqueue + wait), normalise, resample}; the map bucket is the device time of
 * lama_pf_kernel_times (the map update runs asynchronously behind the next scan's sampling). */
int lama_pf_get_summary(lama_pf* h, double ms[4]);
/* uint64_t PFSlam2D::getMemoryUsage() and getMemoryUsage(occmem, dmmem) (src/pf_slam2d.cpp:151-176) from Map::memory() (src/sdm/map.cpp:115-125: per patch
 * 72 bytes of table entry + cell bytes / use count of the shared patch): out = {total over the particles, occmem, dmmem}.  The two-argument overload of the
 * reference adds particle 0's maps P times; occmem / dmmem reproduce that.  On a sharded handle the sums run over this rank's particles.
 * The reference's distance map also owns a patch wherever an occupancy cell was touched; the device counts a distance patch as shared by no more
 * particles than the occupancy patch over the same cells (an upper estimate of the reference's bytes once particles diverge, exact while maps are
 * fully shared). */
int lama_pf_get_memory_usage(lama_pf* h, uint64_t out[3]);
/* const std::deque<double>& PFSlam2D::getTimestamps() (include/lama/pf_slam2d.h:205-206; only the first scan's stamp is ever pushed, src/pf_slam2d.cpp:187) */
int lama_pf_get_timestamps(lama_pf* h, double* stamps, int cap, int* count);
/* work counters of the last update and totals: {residual evals (as the reference would count), ray cells,
   distance-map pops, patches detached, GN iterations, resampled} */
int lama_pf_get_counters(lama_pf* h, uint64_t last[6], uint64_t total[6]);
/* accumulated CUDA-event kernel times in ms {match, raycast, brushfire, resample} and launches {same + misc} */
int lama_pf_kernel_times(lama_pf* h, double ms[4], uint64_t launches[5]);
/* Map::bounds of a particle's map (kind 0 occupancy, 1 distance): min/max cell, *patches = numOfPatches */
int lama_pf_map_bounds(lama_pf* h, int particle, int kind, uint32_t mn[2], uint32_t mx[2], int* patches);
/* Map::write (src/sdm/map.cpp:490-529) of getOccupancyMap(particle) (kind 0) / getDistanceMap(particle) (kind 1): the reference's
 * ".sdm" file -- IOHeader (map.h:95-103), DynamicDistanceMap's max_sqdist_ (dynamic_distance_map.cpp:200-203), then per patch
 * its id, its 1024 cells in the reference cell layout and the 128-byte known mask (container.cpp:143-163). */
int lama_pf_write_map(lama_pf* h, int particle, int kind, const char* path);
/* OccupancyMap::{getProbability, isFree, isOccupied, isUnknown}(Vector3ui) (include/lama/sdm/occupancy_map.h:57-76,
 * frequency_occupancy_map.cpp:110-172) of getOccupancyMap(particle) for n cells: prob[i] = getProbability, flags[i] bit 0 isFree,
 * bit 1 isOccupied, bit 2 isUnknown.  The Vector3d overloads are lama_w2m (Map::w2m, map.h:125-126) followed by this call. */
int lama_pf_occupancy_query(lama_pf* h, int particle, const uint32_t* cells_xy, int n, double* prob, uint8_t* flags);
/* getDistanceMap(particle)->distance(Vector3d, Vector3d* gradient) for n points (distance_map.h:66, dynamic_distance_map.cpp:66-92):
 * dist[n], grad[n][3] (grad may be NULL) */
int lama_pf_distance(lama_pf* h, int particle, const double* pts_xyz, int n, double* dist, double* grad);
int lama_w2m(double resolution, const double* pts_xyz, int n, uint32_t* cells_xy);
/* the grey image sdm::export_to_png encodes (src/sdm/export.cpp:46-96; PFSlam2D::saveOccImage / saveDistImage use it):
 * dims = {width, height} = the map's bounds in cells, pixel (u, v) at pixels[u + v * width]; pixels == NULL only sizes. */
int lama_pf_export_image(lama_pf* h, int particle, int kind, uint8_t* pixels, size_t cap, int dims[2]);
/* dense window of FrequencyOccupancyMap cells {occupied, visited} + Container "known" bit; arrays may be NULL */
int lama_pf_export_occupancy(lama_pf* h, int particle, uint32_t x0, uint32_t y0, int w, int hgt, uint16_t* occupied, uint16_t* visited,
                             uint8_t* known);
/* dense window of DynamicDistanceMap::distance_t fields (dynamic_distance_map.h:48-53) + known bit */
int lama_pf_export_distance(lama_pf* h, int particle, uint32_t x0, uint32_t y0, int w, int hgt, uint16_t* sqdist, uint8_t* valid,
                            uint8_t* known, int16_t* ox, int16_t* oy, uint8_t* queued);

/* ---- multi-GPU behind lama_pf_update: particles shard over shard_count ranks, one host thread / process per GPU.  Rank 0 asks for an
 * id (lama_shard_unique_id = ncclGetUniqueId), hands its 128 bytes to every rank by any means (MPI, a file, torch.distributed ...), and
 * every rank calls lama_pf_shard_connect() on its handle (created with shard_rank / shard_count and the SAME non-zero seed).  From then
 * on lama_pf_update() / lama_pf_update_staged() run the whole sharded step of PFSlam2D::update (src/pf_slam2d.cpp:178-312): match +
 * map update of the local particles (:254-266, :292-302), ONE NCCL all-gather of the match results, normalize / resample (:274-287,
 * :511-574) on identical bytes on every rank, NCCL send / recv of the maps of remote ancestors.  libnccl.so.2 is loaded at run time.
 * lama_pf_shard_stats: {collectives issued, bytes of maps received}. */
int lama_shard_unique_id(uint8_t id[128]);
int lama_pf_shard_connect(lama_pf* h, const uint8_t id[128]);
int lama_pf_shard_stats(lama_pf* h, uint64_t out[2]);

/* --- sharded (multi-GPU) operation: the caller moves the small per-scan vectors between ranks ------------
 * begin : predict (every rank draws the noise of ALL particles, keeping the RNG streams identical) + gate +
 *         scan matching of the local shard; local_out = P_local x 5 doubles (state[4], log-likelihood)
 * finish: takes the gathered P x 5 vector, normalises, decides on resampling and returns the systematic
 *         resampling indices (identical on every rank; rank 0's are broadcast for safety)
 * apply : applies the indices; new local particle k takes the maps of resident slot local_src[k], which is
 *         either a local particle (0 .. P_local-1) or a staging slot (P_local .. 2 P_local-1) previously
 *         filled with lama_pf_particle_unpack from a buffer packed on the ancestor's rank
 * map   : ray-cast + distance-map update of the local shard
 * *did_update of begin: 0 = gated (nothing to do), 1 = first scan handled completely, 2 = matched: the
 * caller must continue with finish [/ apply] / map_update                                                */
int lama_pf_shard_begin(lama_pf* h, const double* pts_xyz, int n, const double sensor_origin[3], const double sensor_quat_xyzw[4],
                        const double odom_xyr[3], double timestamp, int* did_update, double* local_out);
int lama_pf_shard_finish(lama_pf* h, const double* all_results, int* resampled, int32_t* idx);
int lama_pf_shard_apply(lama_pf* h, const int32_t* idx); /* single rank: ancestors are idx themselves */
int lama_pf_shard_apply_local(lama_pf* h, const int32_t* idx, const int32_t* local_src);
int lama_pf_shard_map_update(lama_pf* h);
/* serialise / restore the maps of one resident slot for migration between ranks (host buffers) */
int lama_pf_particle_pack_size(lama_pf* h, int local_particle, size_t* bytes);
int lama_pf_particle_pack(lama_pf* h, int local_particle, void* buf, size_t cap, size_t* used);
int lama_pf_particle_unpack(lama_pf* h, int local_particle, const void* buf, size_t bytes);

/* ------------------------------------------------------------------------------------------------
 * Slam2D -- include/lama/slam2d.h:91-161, src/slam2d.cpp:92-321
 * ------------------------------------------------------------------------------------------------ */
typedef struct lama_slam lama_slam;
typedef struct lama_slam_options { /* Slam2D::Options, slam2d.h:91-125 */
    double trans_thresh, rot_thresh, l2_max, truncated_ray, truncated_range, resolution;
    uint32_t patch_size, max_iter;
    int32_t strategy; /* 0 "gn", 1 "lm" (slam2d.cpp:226-233) */
    int32_t occupancy; /* 0 = FrequencyOccupancyMap as in Slam2D (slam2d.cpp:97); 1 = ProbabilisticOccupancyMap, the log-odds map of
                          src/sdm/probabilistic_occupancy_map.cpp (what LidarOdometry2D pairs with the same update loop) */
    int32_t transient_map;  /* Slam2D::Options::transient_map (slam2d.h:122): after every map update drop the patches that do not
                               meet the (doubled, pose-centred, 2 * maxDistance grown) AABB of the scan, slam2d.cpp:323-379 */
    int32_t lidar_odometry; /* run the handle as lama::LidarOdometry2D (src/lidar_odometry_2d.cpp:42-181): odom_xyr is ignored (may be
                               NULL), log-odds map, l2_max 1.0, rays keep their last metre, map updated after 0.1 m / 0.5 rad of
                               estimated motion, transient map always on; lama_slam_get_pose returns LidarOdometry2D::odom */
    lama_device_options dev;
} lama_slam_options;
int lama_slam_options_default(lama_slam_options* o);
int lama_slam_create(const lama_slam_options* o, lama_slam** out);
int lama_slam_destroy(lama_slam* h);
int lama_slam_set_pose(lama_slam* h, const double xyr[3]);                   /* Slam2D::setPose, slam2d.h:147 */
int lama_slam_update(lama_slam* h, const double* pts_xyz, int n, const double sensor_origin[3], const double sensor_quat_xyzw[4],
                     const double odom_xyr[3], double timestamp, int* did_update); /* Slam2D::update, slam2d.cpp:143-198 */
int lama_slam_get_pose(lama_slam* h, double xyr[3]);
int lama_slam_get_state(lama_slam* h, double state[4]);
int lama_slam_get_processed_cells(lama_slam* h, uint32_t* n);               /* getNumberOfProcessedCells, slam2d.h:139 */
int lama_slam_get_map_stats(lama_slam* h, uint64_t stats[2]);                /* {map updates so far, patches deleted by the transient map} */
int lama_slam_get_counters(lama_slam* h, uint64_t last[6], uint64_t total[6]);
int lama_slam_kernel_times(lama_slam* h, double ms[4], uint64_t launches[5]);
int lama_slam_map_bounds(lama_slam* h, int kind, uint32_t mn[2], uint32_t mx[2], int* patches);
int lama_slam_export_occupancy(lama_slam* h, uint32_t x0, uint32_t y0, int w, int hgt, uint16_t* occupied, uint16_t* visited, uint8_t* known);
/* occupancy == 1 only: dense window of ProbabilisticOccupancyMap cells (float log-odds, prob_tag) + Container known bit */
int lama_slam_occupancy_query(lama_slam* h, const uint32_t* cells_xy, int n, double* prob, uint8_t* flags);   /* as lama_pf_occupancy_query */
int lama_slam_distance(lama_slam* h, const double* pts_xyz, int n, double* dist, double* grad);                  /* as lama_pf_distance */
int lama_slam_write_map(lama_slam* h, int kind, const char* path);                                     /* as lama_pf_write_map */
int lama_slam_export_image(lama_slam* h, int kind, uint8_t* pixels, size_t cap, int dims[2]);           /* as lama_pf_export_image */
int lama_slam_export_logodds(lama_slam* h, uint32_t x0, uint32_t y0, int w, int hgt, float* logodds, uint8_t* known);
int lama_slam_export_distance(lama_slam* h, uint32_t x0, uint32_t y0, int w, int hgt, uint16_t* sqdist, uint8_t* valid, uint8_t* known,
                              int16_t* ox, int16_t* oy, uint8_t* queued);

/* ------------------------------------------------------------------------------------------------
 * Loc2D (match path) -- include/lama/loc2d.h:59-130, src/loc2d.cpp:46-192
 * The caller fills the public distance_map (loc2d.h:104) through the lama_dm_* grid interface.
 * ------------------------------------------------------------------------------------------------ */
typedef struct lama_loc lama_loc;
typedef struct lama_dm lama_dm; /* a device-resident DynamicDistanceMap */
typedef struct lama_loc_options { /* Loc2D::Options, loc2d.cpp:46-58 */
    double trans_thresh, rot_thresh, l2_max, resolution;
    uint32_t patch_size, max_iter;
    int32_t strategy;
    uint32_t gloc_particles, gloc_iters; /* globalLocalization: candidates per attempt, attempts (loc2d.cpp:53-54) */
    double gloc_thresh;                  /* RMSE that ends global localisation (loc2d.cpp:55) */
    double cov_blend;                    /* blend of the sampling covariance into the solver covariance (loc2d.cpp:57,199-247) */
    double center_xy[2]; /* where to centre the device map window */
    lama_device_options dev;
} lama_loc_options;
int lama_loc_options_default(lama_loc_options* o);
int lama_loc_create(const lama_loc_options* o, lama_loc** out);              /* Loc2D::Init, loc2d.cpp:61-108 */
int lama_loc_destroy(lama_loc* h);
int lama_loc_distance_map(lama_loc* h, lama_dm** dm);                        /* borrowed: Loc2D::distance_map */
int lama_loc_set_pose(lama_loc* h, const double xyr[3]);                     /* Loc2D::setPose, loc2d.h:117-118 */
int lama_loc_update(lama_loc* h, const double* pts_xyz, int n, const double sensor_origin[3], const double sensor_quat_xyzw[4],
                    const double odom_xyr[3], double timestamp, int force_update, int* did_update); /* loc2d.cpp:126-192 */
int lama_loc_get_pose(lama_loc* h, double xyr[3]);
int lama_loc_get_state(lama_loc* h, double state[4]);
int lama_loc_get_covar(lama_loc* h, double cov[9]);                          /* Loc2D::getCovar */
int lama_loc_get_rmse(lama_loc* h, double* rmse);                            /* Loc2D::getRMSE */
int lama_loc_get_solve_stats(lama_loc* h, uint32_t stats[2]);                /* {iterations, residual evaluations} */
/* public `occupancy_map` (SimpleOccupancyMap, loc2d.h:103): setFree (state -1) / setUnknown (0) / setOccupied (1) on n cells */
int lama_loc_occupancy_set(lama_loc* h, const uint32_t* cells_xy, int n, int state);
int lama_loc_occupancy_read(lama_loc* h, const char* path);                   /* occupancy_map->read(file): SimpleOccupancyMap, Map::read map.cpp:531-575 */
int lama_loc_set_seed(lama_loc* h, uint32_t seed);                            /* random::setSeed for the sampling below */
int lama_loc_trigger_global_localization(lama_loc* h);                        /* Loc2D::triggerGlobalLocalization, loc2d.cpp:194-197 */
int lama_loc_global_localization_active(lama_loc* h, int* active);

/* ------------------------------------------------------------------------------------------------
 * SDM grid interface on a device-resident DynamicDistanceMap
 * include/lama/sdm/distance_map.h:66-70, dynamic_distance_map.h:55-66
 * ------------------------------------------------------------------------------------------------ */
int lama_dm_create(double resolution, uint32_t patch_size, double l2_max, const double center_xy[2], const lama_device_options* dev, lama_dm** out);
int lama_dm_destroy(lama_dm* dm);
int lama_dm_max_sqdist(lama_dm* dm, uint32_t* max_sqdist);
/* addObstacle / removeObstacle on n cells in list order, dynamic_distance_map.cpp:212-242; nothing propagates until update */
int lama_dm_add_obstacles(lama_dm* dm, const uint32_t* cells_xy, int n);
int lama_dm_remove_obstacles(lama_dm* dm, const uint32_t* cells_xy, int n);
/* DynamicDistanceMap::update(), dynamic_distance_map.cpp:160-197; *processed = its return value */
int lama_dm_update(lama_dm* dm, uint32_t* processed);
/* DistanceMap::distance(Vector3d, Vector3d* grad) for n points; grad (n x 3) may be NULL */
int lama_dm_distance(lama_dm* dm, const double* pts_xyz, int n, double* dist, double* grad);
int lama_dm_bounds(lama_dm* dm, uint32_t mn[2], uint32_t mx[2], int* patches);
int lama_dm_write(lama_dm* dm, const char* path);   /* Map::write, map.cpp:490-529 */
int lama_dm_read(lama_dm* dm, const char* path);    /* Map::read, map.cpp:531-575, into an empty map of the same resolution and l2_max */
int lama_dm_export_image(lama_dm* dm, uint8_t* pixels, size_t cap, int dims[2]);   /* sdm::export_to_png(DistanceMap), export.cpp:75-96 */
int lama_dm_export(lama_dm* dm, uint32_t x0, uint32_t y0, int w, int hgt, uint16_t* sqdist, uint8_t* valid, uint8_t* known, int16_t* ox,
                   int16_t* oy, uint8_t* queued);
/* upload distance_t fields for a patch-aligned window (x0, y0, w, hgt multiples of 32); cells with known == 0 are left absent */
int lama_dm_import(lama_dm* dm, uint32_t x0, uint32_t y0, int w, int hgt, const uint16_t* sqdist, const uint8_t* valid, const uint8_t* known,
                   const int16_t* ox, const int16_t* oy, const uint8_t* queued);

/* Solver plug point: the weighted normal equations of MatchSurface2D at `count` SE2 states on one distance
 * map, so that a host nlls::Strategy (nlls/strategy.h:43-82) can drive the device evaluation.
 * out = count x 12: {A00,A01,A02,A11,A12,A22, g0,g1,g2, chi2, sum d^2, sum -d^2/meas_sigma} */
int lama_dm_match_normal_equations(lama_dm* dm, const double* pts_xyz, int n, const double sensor_origin[3], const double sensor_quat_xyzw[4],
                                   const double* states, int count, int robust_kind, double robust_param, double meas_sigma, double* out);
/* Solve(options, MatchSurface2D, cov) for `count` start states (nlls/solver.h:84); states updated in place;
 * stats = count x 2 {iterations, evaluations}; sums = count x 12 at the final states (may be NULL) */
int lama_dm_match_solve(lama_dm* dm, const double* pts_xyz, int n, const double sensor_origin[3], const double sensor_quat_xyzw[4], double* states,
                        int count, int strategy, int robust_kind, double robust_param, uint32_t max_iter, uint32_t* stats, double* sums);

/* MatchSurface2D::error() (src/match_surface_2d.cpp:92-116): sqrt(sum d^2 / N), d = nearest-cell distance, of the cloud at `count` states */
int lama_dm_match_error(lama_dm* dm, const double* pts_xyz, int n, const double sensor_origin[3], const double sensor_quat_xyzw[4], const double* states, int count,
                        double* rmse);

/* ---- lama::SimplePGO::optimize (include/lama/simple_pgo.h:43-57, src/simple_pgo.cpp:48-105): pose-graph optimisation on the device ----
 * nodes_xyr = node_list (n_nodes x {x, y, rotation}), edges = edge_list (from, to pairs + measured relative poses), fixed = fixed_list.
 * The factor graph is the reference's: a prior on node 0 (sigmas 1) or on every fixed node (sigmas 0.1), BetweenFactor<SE2> on consecutive
 * nodes (measured = node[i]^-1 node[i+1]) and on the edges, sigmas (0.5, 0.5, 0.1), miniSAM Levenberg-Marquardt with diagonal damping
 * (vendor/minisam/minisam/nonlinear/LevenbergMarquardtOptimizer.cpp:56-332).  *status = miniSAM's NonlinearOptimizationStatus (0 SUCCESS,
 * 1 MAX_ITERATION, 2 ERROR_INCREASE, 3 RANK_DEFICIENCY, 4 INVALID); like the reference, nodes_xyr is only updated on SUCCESS.
 * report = {LM iterations, lambda tries, CG iterations, initial error, final error, device ms}. */
int lama_pgo_optimize(int device, double* nodes_xyr, int n_nodes, const int* edges_from_to, const double* edges_xyr, int n_edges, const int* fixed_nodes,
                      const double* fixed_xyr, int n_fixed, int* status, double report[6]);

/* ---- GraphSlam2D's loop-closure front end on a device map (src/graph_slam2d.cpp:283-392) ----
 * findLoopClosureCandidates (:283-313): ids of the key poses (x, y pairs) within `radius` of the query among the first
 * n_keys - ignore_n_chain_poses, nearest first, at most max_candidates (Options::loop_max_candidates, graph_slam2d.h:75). */
int lama_loop_closure_candidates(const double* key_xy, int n_keys, int ignore_n_chain_poses, const double query_xy[2], double radius, int max_candidates, int* ids,
                                 int* count);
/* correlateCandidateScan (:315-355): the candidate key pose's cloud against the distance map -- one Gauss-Newton iteration (Huber 0.15) from
 * the candidate's pose and one from the reference position, the better start refined to convergence; between = matched pose - ref pose
 * (Pose2D::operator-, pose2d.cpp:81-84), *rmse = MatchSurface2D::error() there.  ref / cand poses are the corrected key poses (:319-320). */
int lama_slam_correlate_candidate_scan(lama_slam* h, const double* pts_xyz, int n, const double sensor_origin[3], const double sensor_quat_xyzw[4],
                                       const double ref_xyr[3], const double cand_xyr[3], double between_xyr[3], double* rmse);
int lama_dm_correlate_candidate_scan(lama_dm* dm, const double* pts_xyz, int n, const double sensor_origin[3], const double sensor_quat_xyzw[4],
                                     const double ref_xyr[3], const double cand_xyr[3], double between_xyr[3], double* rmse);
/* coarseSearchAndCorrelateCandidateScan (:357-392): first against a coarse distance map (0.25 m cells, 2.5 m reach) built from the reference
 * key pose's cloud alone, then against the map itself. */
int lama_slam_coarse_correlate_candidate_scan(lama_slam* h, const double* ref_pts_xyz, int ref_n, const double ref_origin[3], const double ref_quat_xyzw[4],
                                              const double* pts_xyz, int n, const double sensor_origin[3], const double sensor_quat_xyzw[4],
                                              const double ref_xyr[3], const double cand_xyr[3], double between_xyr[3], double* rmse);
int lama_dm_coarse_correlate_candidate_scan(lama_dm* dm, const double* ref_pts_xyz, int ref_n, const double ref_origin[3], const double ref_quat_xyzw[4],
                                            const double* pts_xyz, int n, const double sensor_origin[3], const double sensor_quat_xyzw[4],
                                            const double ref_xyr[3], const double cand_xyr[3], double between_xyr[3], double* rmse);

/* ---- miniSAM Levenberg-Marquardt over an explicit SE2 factor graph (vendor/minisam/minisam/nonlinear/LevenbergMarquardtOptimizer.cpp:56-332) ----
 * priors: PriorFactor<SE2> on prior_nodes[i] measured prior_xyr[i]; betweens: BetweenFactor<SE2> between_from_to[2i] -> [2i+1] measured between_xyr[i].
 * Each factor's loss is loss[4] = {sigma_x, sigma_y, sigma_theta, huber_k}: huber_k <= 0 gives DiagonalLoss::Sigmas (core/LossFunction.cpp:95-114),
 * huber_k > 0 gives HuberLoss::Huber(huber_k) on the raw error (:190-203; the sigmas are ignored).  Factors enter the graph priors first, then
 * betweens, in the given order.  *status, report and the SUCCESS-only update of nodes_xyr are those of lama_pgo_optimize.  accepted (may be NULL)
 * receives one byte per tried lambda, 1 accepted / 0 rejected, at most accepted_cap of them; *n_tries (may be NULL) = the number of tries. */
int lama_pgo_optimize_graph(int device, double* nodes_xyr, int n_nodes, const int* prior_nodes, const double* prior_xyr, const double* prior_loss, int n_priors,
                            const int* between_from_to, const double* between_xyr, const double* between_loss, int n_betweens, int* status, double report[6],
                            uint8_t* accepted, int accepted_cap, int* n_tries);

/* ------------------------------------------------------------------------------------------------
 * GraphSlam2D -- include/lama/graph_slam2d.h:51-173, src/graph_slam2d.cpp:104-430: key-pose graph SLAM over a transient-map Slam2D,
 * loop closures by scan correlation against the local map, Huber-robust pose-graph optimisation on the device.
 * ------------------------------------------------------------------------------------------------ */
typedef struct lama_graph lama_graph;
typedef struct lama_graph_options { /* GraphSlam2D::Options, graph_slam2d.h:59-87 */
    lama_slam_options slam;            /* transient_map and truncated_ray are forced to 1 and 1.0 (graph_slam2d.cpp:106-107) */
    double key_pose_distance;          /* linear distance between key poses */
    double key_pose_angular_distance;  /* angular distance between key poses */
    int32_t key_pose_head_delay;       /* the loop search queries the key pose this many keys back */
    double loop_search_max_distance;   /* search radius max^r min^(1 - r), r = min(accumulated distance, 100) / 100 */
    double loop_search_min_distance;
    int32_t loop_max_candidates;       /* candidates correlated per search */
    double loop_closure_scan_rmse;     /* largest correlation RMSE accepted (twice that after the coarse retry) */
    int32_t loop_closure_max_candidates; /* declared but unused by the reference; accepted and ignored */
    int32_t ignore_n_chain_poses;      /* the newest key poses left out of the search */
} lama_graph_options;
/* the reference defaults: Slam2D's (lama_slam_options_default) and graph_slam2d.h:62-86 */
int lama_graph_options_default(lama_graph_options* o);
int lama_graph_create(const lama_graph_options* o, lama_graph** out);   /* GraphSlam2D::GraphSlam2D, graph_slam2d.cpp:104-111 */
int lama_graph_destroy(lama_graph* h);
int lama_graph_set_pose(lama_graph* h, const double xyr[3]);             /* GraphSlam2D::Init, graph_slam2d.cpp:118-121 */
/* bool GraphSlam2D::update(surface, odometry, timestamp), graph_slam2d.cpp:188-282; *did_update = the bool (may be NULL) */
int lama_graph_update(lama_graph* h, const double* pts_xyz, int n, const double sensor_origin[3], const double sensor_quat_xyzw[4],
                      const double odom_xyr[3], double timestamp, int* did_update);
int lama_graph_get_pose(lama_graph* h, double xyr[3]);                   /* GraphSlam2D::getPose = correction + slam pose, :127-129 */
/* key_poses: corrected[cap x 3], original[cap x 3], stamps[cap] (each may be NULL); *count = number of key poses (cap = capacity) */
int lama_graph_get_key_poses(lama_graph* h, double* corrected_xyr, double* original_xyr, double* stamps, int cap, int* count);
/* the cloud of key pose `key` (its sensor origin / quaternion may be NULL): n x 3 points, *count = n */
int lama_graph_get_key_cloud(lama_graph* h, int key, double* pts_xyz, int cap, double sensor_origin[3], double sensor_quat_xyzw[4], int* count);
/* links (graph_slam2d.h:116-117): cap x {candidate key, reference key}, *count = number of links */
int lama_graph_get_links(lama_graph* h, int32_t* from_to, int cap, int* count);
/* the candidate ids of the latest update's loop search, nearest first (*count = 0 when that update did not search) */
int lama_graph_get_last_candidates(lama_graph* h, int32_t* ids, int cap, int* count);
/* counts[4] = {key poses, loop factors, optimisations run, optimisations that ended in SUCCESS}; last_status and last_report (as
 * lama_pgo_optimize's) describe the latest optimisation (status -1 before the first); either output may be NULL */
int lama_graph_get_stats(lama_graph* h, uint64_t counts[4], int* last_status, double last_report[6]);
/* the inner Slam2D (GraphSlam2D::slam) as a BORROWED handle: the lama_slam_* getters, exports and map writers work on the local map;
 * lama_slam_destroy on it does nothing, and it dies with the lama_graph */
int lama_graph_slam(lama_graph* h, lama_slam** slam);

/* ------------------------------------------------------------------------------------------------
 * FrequencyOccupancyMap -- include/lama/sdm/frequency_occupancy_map.h: a device-resident {occupied, visited} map with its own
 * 'known' plane (a pruned cell is {0, 0} and still known).  Cells outside the directory window make a call fail with
 * LAMA_ERR_WINDOW; the map is then partly updated.
 * ------------------------------------------------------------------------------------------------ */
typedef struct lama_om lama_om;
/* FrequencyOccupancyMap(resolution, patch_size), window of dev->dir_dim^2 patches centred on center_xy (NULL: origin); dev->pool_slots
 * 0 = dir_dim^2 patches, so a full window cannot run out */
int lama_om_create(double resolution, uint32_t patch_size, const double center_xy[2], const lama_device_options* dev, lama_om** out);
int lama_om_destroy(lama_om* om);   /* does nothing on a borrowed handle */
/* the loop of GraphSlam2D::generateOccupancyMap (graph_slam2d.cpp:135-160) for any posed scans: scan k = points [offsets[k],
 * offsets[k + 1]) of pts_xyz (offsets[0] = 0), sensor origins + 3k / quats_xyzw + 4k (either may be NULL: identity), base pose
 * states + 4k as SE2 {cos, sin, x, y}.  In point order: setOccupied(tf * p), and with `full` setFree on every cell of
 * computeRay(w2m(tf.translation()), w2m(tf * p)) (both ends excluded).  *cells (may be NULL) = cell updates.  No prune. */
int lama_om_insert_scans(lama_om* om, const double* pts_xyz, const int64_t* offsets, int n_scans, const double* origins, const double* quats_xyzw,
                         const double* states, int full, uint64_t* cells);
int lama_om_prune(lama_om* om);   /* FrequencyOccupancyMap::prune, frequency_occupancy_map.cpp:149-158 */
int lama_om_resolution(lama_om* om, double* resolution);
int lama_om_bounds(lama_om* om, uint32_t mn[2], uint32_t mx[2], int* patches);   /* Map::bounds in cells, map.cpp:139-157 */
/* flags bit 0 isFree, bit 1 isOccupied, bit 2 isUnknown; prob = getProbability (as lama_pf_occupancy_query) */
int lama_om_query(lama_om* om, const uint32_t* cells_xy, int n, double* prob, uint8_t* flags);
int lama_om_export(lama_om* om, uint32_t x0, uint32_t y0, int w, int hgt, uint16_t* occupied, uint16_t* visited, uint8_t* known);
int lama_om_write(lama_om* om, const char* path);                                   /* Map::write, map.cpp:490-529 */
int lama_om_export_image(lama_om* om, uint8_t* pixels, size_t cap, int dims[2]);   /* sdm::export_to_png(OccupancyMap), export.cpp:46-73 */
/* with dev->timing: ms[1] = device time of the casts (lama_om_insert_scans), launches as lama_slam_kernel_times */
int lama_om_kernel_times(lama_om* om, double ms[4], uint64_t launches[5]);
/* GraphSlam2D::generateOccupancyMap(full) (graph_slam2d.cpp:131-164): after an optimisation (or on the first call) a new map at
 * (full ? resolution : 0.1 m), then the key scans not yet cast, at their corrected poses, then prune over the whole map.  The handle
 * is BORROWED: owned by the lama_graph, and the map behind it is replaced in place when it is recreated (possibly at another
 * resolution), where the reference hands out a new shared_ptr. */
int lama_graph_generate_occupancy_map(lama_graph* h, int full, lama_om** om);
/* GraphSlam2D::generateCoarseDistanceMap (graph_slam2d.cpp:166-186): a new 0.1 m distance map with a 5 m reach and an obstacle at
 * every occupied cell of the inner Slam2D, visited in ascending directory index, then cell index (x fastest); *processed (may be
 * NULL) = its update() return value.  BORROWED like the occupancy map. */
int lama_graph_generate_coarse_distance_map(lama_graph* h, lama_dm** dm, uint32_t* processed);

/* ------------------------------------------------------------------------------------------------
 * TruncatedSignedDistanceMap -- include/lama/sdm/truncated_signed_distance_map.h, src/sdm/truncated_signed_distance_map.cpp:
 * cells {float distance; float weight} and an "on" bit, in a dense window of window[0] x window[1] x window[2] patches of 32 x 32
 * (x 32 in 3-D) cells.  Cells are absolute map coordinates (x, y, z) as Map::w2m gives them; in 2-D, z is not addressed.
 * ------------------------------------------------------------------------------------------------ */
typedef struct lama_tsdm lama_tsdm;
/* TruncatedSignedDistanceMap(resolution, patch_size, is3d) (:41-49); patch_size must be 32.  The window is centred on center_xyz
 * (NULL: origin); window_patches NULL = (dev->dir_dim, dev->dir_dim, 1) in 2-D and (8, 8, 4) in 3-D, at most 2048 per axis.
 * dev->pool_slots 0 = one patch per window entry (a 3-D patch is 260 KiB, so the 3-D default takes 65 MiB). */
int lama_tsdm_create(double resolution, uint32_t patch_size, int is3d, const double center_xyz[3], const int32_t window_patches[3],
                     const lama_device_options* dev, lama_tsdm** out);
int lama_tsdm_destroy(lama_tsdm* h);
int lama_tsdm_set_max_distance(lama_tsdm* h, double distance);   /* setMaxDistance (:210-213): truncate_size_ */
int lama_tsdm_max_distance(lama_tsdm* h, double* distance);      /* maxDistance (:215-218) */
/* n_clouds calls of insertPointCloud (:141-158) in order: cloud k = points [offsets[k], offsets[k + 1]) of pts_xyz (offsets[0] = 0),
 * sensor origins + 3k / quats_xyzw + 4k in world coordinates (either may be NULL: zero / identity); inserted[k] (may be NULL) = its
 * return value, the number of distinct hit cells.  A hit or a ray cell outside the window fails with LAMA_ERR_WINDOW (in 2-D also a
 * hit more than 2^15 cells from world z = 0), a full pool with LAMA_ERR_POOL; the map is then unchanged. */
int lama_tsdm_insert_point_clouds(lama_tsdm* h, const double* pts_xyz, const int64_t* offsets, int n_clouds, const double* origins,
                                  const double* quats_xyzw, uint64_t* inserted);
/* distance(Vector3d, gradient) (:59-130) of n world points: bilinear in 2-D, trilinear in 3-D; gradient (n x 3) may be NULL */
int lama_tsdm_distance(lama_tsdm* h, const double* pts_xyz, int n, double* distance, double* gradient);
/* Map::bounds (map.cpp:139-157) in cells, all three axes; *patches (may be NULL) = allocated patches */
int lama_tsdm_bounds(lama_tsdm* h, uint32_t mn[3], uint32_t mx[3], int* patches);
/* the cells of the box lo + [0, size) (x fastest, then y, then z); cells that are off read 0; any output may be NULL */
int lama_tsdm_export(lama_tsdm* h, const uint32_t lo[3], const int32_t size[3], float* distance, float* weight, uint8_t* on);
/* toMesh (:220-272): 3 unshared vertices (x, y, z floats) per triangle, PolygonMesh::index[i] = i.  *n_vertices = the vertex count;
 * the vertices are written when vertices != NULL and cap (in vertices) >= *n_vertices.  Cells are visited in ascending window
 * entry, then cell index, where the reference iterates an unordered_map. */
int lama_tsdm_to_mesh(lama_tsdm* h, float* vertices, size_t cap, size_t* n_vertices);
/* sdm::export_to_ply (export.cpp:112-143): ASCII PLY of toMesh, faces written as 3 i+2 i+1 i */
int lama_tsdm_write_ply(lama_tsdm* h, const char* path);
/* with dev->timing: ms = device time of [0] insert_point_clouds, [1] distance, [2] to_mesh; launches likewise */
int lama_tsdm_kernel_times(lama_tsdm* h, double ms[3], uint64_t launches[3]);

/* ------------------------------------------------------------------------------------------------
 * 3-D occupancy maps -- FrequencyOccupancyMap / ProbabilisticOccupancyMap(resolution, patch_size, is3d = true)
 * (include/lama/sdm/frequency_occupancy_map.h, probabilistic_occupancy_map.h, src/sdm/map.cpp:42-48): cells {uint16 occupied;
 * uint16 visited} (kind 0, frequency) or a float log-odds (kind 1), and a known bit, in a dense window of window[0] x window[1] x
 * window[2] patches of 32 x 32 x 32 cells.  Cells are absolute map coordinates (x, y, z) as Map::w2m gives them (lama_w2m3).
 * ------------------------------------------------------------------------------------------------ */
typedef struct lama_om3 lama_om3;
/* ops of lama_om3_apply */
#define LAMA_OM3_SET_FREE 0
#define LAMA_OM3_SET_OCCUPIED 1
#define LAMA_OM3_SET_UNKNOWN 2
/* the map of `kind` (0 frequency, 1 log-odds) with is3d = true; patch_size must be 32.  The window is centred on center_xyz (NULL:
 * origin); window_patches NULL = (8, 8, 4), at most 2048 per axis and 65 536 entries in all.  dev->pool_slots 0 = one patch per
 * window entry (a patch is 132 KiB, so the default takes 33 MiB). */
int lama_om3_create(double resolution, uint32_t patch_size, int kind, const double center_xyz[3], const int32_t window_patches[3],
                    const lama_device_options* dev, lama_om3** out);
int lama_om3_destroy(lama_om3* h);
/* the loop body of GraphSlam2D::generateOccupancyMap (graph_slam2d.cpp:146-158) for every point of n_clouds clouds in order:
 * setOccupied(tf * p), then with `full` setFree on computeRay(w2m(tf.translation()), w2m(tf * p)), tf = Translation(origin) * quat.
 * Clouds as lama_tsdm_insert_point_clouds.  *cells (may be NULL) = the cell updates made.  A cell outside the window fails with
 * LAMA_ERR_WINDOW, a full pool with LAMA_ERR_POOL; the map is then unchanged. */
int lama_om3_insert_point_clouds(lama_om3* h, const double* pts_xyz, const int64_t* offsets, int n_clouds, const double* origins,
                                 const double* quats_xyzw, int full, uint64_t* cells);
/* setFree / setOccupied / setUnknown (LAMA_OM3_SET_*) of n cells in list order (frequency_occupancy_map.cpp:65-108,
 * probabilistic_occupancy_map.cpp:82-123); changed[i] (may be NULL) = what op i returns.  Errors as insert. */
int lama_om3_apply(lama_om3* h, const uint32_t* cells_xyz, const uint8_t* ops, int n, uint8_t* changed);
/* getProbability (prob, may be NULL) and flags (may be NULL) bit 0 isFree, bit 1 isOccupied, bit 2 isUnknown of n cells */
int lama_om3_query(lama_om3* h, const uint32_t* cells_xyz, int n, double* prob, uint8_t* flags);
/* FrequencyOccupancyMap::prune (frequency_occupancy_map.cpp:149-158); LAMA_ERR_ARG on a log-odds map */
int lama_om3_prune(lama_om3* h);
/* Map::bounds (map.cpp:139-157) in cells, all three axes; *patches (may be NULL) = allocated patches */
int lama_om3_bounds(lama_om3* h, uint32_t mn[3], uint32_t mx[3], int* patches);
/* the box lo + [0, size) (x fastest, then y, then z): cell words ({occupied | visited << 16} or the float bits) and known bits;
 * either output may be NULL */
int lama_om3_export(lama_om3* h, const uint32_t lo[3], const int32_t size[3], uint32_t* cells, uint8_t* known);
/* Map::write (map.cpp:490-529) with is_3d = 1: patches in ascending window entry, where the reference iterates an unordered_map */
int lama_om3_write(lama_om3* h, const char* path);
/* Map::read (map.cpp:531-575) into an empty map: a 4-byte-cell 3-D file, whose resolution the map takes */
int lama_om3_read(lama_om3* h, const char* path);
/* the z-slice image of sdm::export_to_png(occ, file, zed) (export.cpp:46-72): dims = {width, height} from the x / y bounds, slice
 * z = w2m((0, 0, zed)).z; pixels (row-major, width per row) written when cap >= width * height */
int lama_om3_export_image(lama_om3* h, double zed, uint8_t* pixels, size_t cap, int dims[2]);
/* with dev->timing: ms = device time of [0] insert_point_clouds, [1] apply, [2] query; launches likewise */
int lama_om3_kernel_times(lama_om3* h, double ms[3], uint64_t launches[3]);
/* Map::w2m (map.h:125-126) on all three axes: world points (n x 3) -> cells (n x 3) */
int lama_w2m3(double resolution, const double* pts_xyz, int n, uint32_t* cells_xyz);

/* ------------------------------------------------------------------------------------------------
 * Checkpoints (no counterpart in the reference): save a PFSlam2D, Slam2D or GraphSlam2D session to a file and continue it later, in
 * another process or on another device, bit for bit as if it had not stopped.  The file holds the options, the front end's state (poses,
 * weights, trajectories, the mt19937 state, counters, the Summary buckets) and the device maps with their copy-on-write sharing;
 * a GraphSlam2D file also holds its key poses with their clouds, links, pose graph, loop-factor queue and correction, the inner Slam2D
 * and the global occupancy map when the next lama_graph_generate_occupancy_map would add to it (the coarse distance map is rebuilt by
 * every call and is not saved).  DESIGN.md section 13 gives the layout.  Saving settles the pending map update first and does not
 * change the handle.  Kernel times,
 * traffic counters and staged scans start empty on a loaded handle (lama_pf_update_staged needs a new lama_pf_stage_scans).
 * Loading checks the whole file (size, checksum, version, kind, every count, directory entry and reference count) before it touches
 * CUDA: a bad file gives LAMA_ERR_ARG and no handle; a valid file on a host without a device gives LAMA_ERR_NO_DEVICE.
 * From `dev` (may be NULL: device 0) only device, stream and timing are taken; dir_dim, pool_slots and max_beams must be 0 or the
 * saved values.  A sharded PFSlam2D (shard_count > 1) cannot be saved (LAMA_ERR_STATE).  A LidarOdometry2D-mode Slam2D loads back in
 * that mode.  Each loader refuses the other kinds' files (LAMA_ERR_ARG); the inner Slam2D of a lama_graph (lama_graph_slam) can still
 * be saved on its own and loads back as a standalone Slam2D.
 * ------------------------------------------------------------------------------------------------ */
int lama_pf_save_state(lama_pf* h, const char* path);
int lama_pf_load_state(const char* path, const lama_device_options* dev, lama_pf** out);
int lama_slam_save_state(lama_slam* h, const char* path);
int lama_slam_load_state(const char* path, const lama_device_options* dev, lama_slam** out);
int lama_graph_save_state(lama_graph* h, const char* path);
int lama_graph_load_state(const char* path, const lama_device_options* dev, lama_graph** out);
/* what the last save or load on this thread took and moved.  ms = {count, compaction, gather (device, CUDA events; save only), slot
 * copy (chunked through pinned buffers), engine creation, tables (directories, reference counts, free stack; load only), encode
 * (serialisation / parsing, checks and checksum), file I/O, total}; sizes = {slots in use, per-particle patch references, file bytes}.
 * For a GraphSlam2D, device times, slots and references are the sums over its two engines (inner Slam2D and global map). */
int lama_checkpoint_last_stats(double ms[9], uint64_t sizes[3]);

#ifdef __cplusplus
}
#endif
#endif /* LAMA_B200_H */
