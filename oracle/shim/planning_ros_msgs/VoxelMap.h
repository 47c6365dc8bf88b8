/* Stand-in for the generated planning_ros_msgs/VoxelMap.h (TEST INFRASTRUCTURE): the fields of planning_ros_msgs/msg/
 * VoxelMap.msg that voxel_grid.cpp writes — geometry_msgs/Point origin and dim, float32 resolution,
 * int8[] data.  The header is not written by VoxelGrid and is left out. */
#ifndef MPLB_SHIM_PLANNING_ROS_MSGS_VOXELMAP
#define MPLB_SHIM_PLANNING_ROS_MSGS_VOXELMAP
#include <cstdint>
#include <vector>
namespace planning_ros_msgs {
struct VoxelMap {
  struct { double x, y, z; } origin, dim;
  float resolution;
  std::vector<int8_t> data;
};
}  // namespace planning_ros_msgs
#endif
