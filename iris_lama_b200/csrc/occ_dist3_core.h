// occ_dist3_core.h -- the per-cell filter of the coupled insertion (OccMap3Dev::insert_point_clouds_dm3, om3d.cu), shared with the
// host emulation (tests/emu/occ_dist3_emu.cpp).  Plain C++ usable from host and device.
//
// The reference couples an occupancy map to its distance map through the setters' return values (slam2d.cpp:271-316,
// pf_slam2d.cpp:439-509): `if (occupancy_map_->setOccupied(c)) distance_map_->addObstacle(c)`, then along the ray `if
// (occupancy_map_->setFree(c)) distance_map_->removeObstacle(c)`, and update() once per cloud.  Such a setter call that returns true is
// an event.  Every event does the mutable Map::get of addObstacle / removeObstacle (allocate the patch, set the known bit), which does
// not depend on order.  It pushes a heap entry only when it changes whether the cell is an obstacle (valid && sqdist == 0): an add on a
// cell that is not one, a remove on one that is (dynamic_distance_map.cpp:212-242).  Nothing else changes that state: raise()
// invalidates only cells whose obstacle is invalid, and an obstacle is its own obstacle (:244-279); lower() writes sqdist >= 1 only,
// because it never writes in the direction of the cell's obstacle (:296).  So the thread that folds one cell's records in record order
// can start from the distance-map cell as the previous ops left it and decide every push of that cell.
#pragma once

#include "ddm3_core.h"
#include "om3d_core.h"

namespace lama_b200 {

// per-record flags
enum : uint32_t { kOd3Event = 1u, kOd3Push = 2u, kOd3Remove = 4u };

LAMA_HD bool dm3_obstacle(uint64_t c) { return dm3_valid(c) && dm3_sqdist(c) == 0; }

// One record of a cell's run, in record order: r = op in bits 0-1 (kOm3SetOccupied or kOm3SetFree).  Folds the setter into the
// occupancy word and returns 0 (it returned false) or kOd3Event, with kOd3Remove for a setFree and kOd3Push when the distance-map op
// pushes; `obstacle` is the distance-map cell's state and follows the ops.
LAMA_HD uint32_t od3_record(int kind, const ProbParams& pp, uint32_t& word, uint32_t r, bool& obstacle)
{
    const uint32_t op = r & 3u;
    if (!om3_op(kind, word, op, pp)) return 0u;
    const bool add = op == kOm3SetOccupied;
    const uint32_t ev = kOd3Event | (add ? 0u : kOd3Remove);
    if (add == obstacle) return ev;   // addObstacle on an obstacle, removeObstacle on a non-obstacle: only the get()
    obstacle = add;
    return ev | kOd3Push;
}

}  // namespace lama_b200
