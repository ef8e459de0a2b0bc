// Stand-in for ros/ros.h in oracle/_ref/libfuel_ref_tour.so: the tick clock of ../../ref_standin_view/ros/ros.h, plus
// what exploration_manager/src/fast_exploration_manager.cpp uses beyond it: ROS_ERROR_COND and a string parameter.
// TEST INFRASTRUCTURE ONLY.
#pragma once
#include "../../ref_standin_view/ros/ros.h"

#define ROS_ERROR_COND(...) do {} while (0)

namespace ros {
template <>
inline bool NodeHandle::param<std::string>(const std::string& key, std::string& out, const std::string& def) const {
  out = def;
  return false;
}
}  // namespace ros
