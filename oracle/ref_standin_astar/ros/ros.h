// Stand-in for ros/ros.h as path_searching/src/astar2.cpp and the plan_env headers use it: the facilities of
// ../../ref_standin/ros/ros.h (NodeHandle::param fed from a table, silent log macros) with a tick clock.  Every
// ros::Time::now() advances the clock by one second, and Astar::search calls it once before its loop and once per loop
// iteration (astar2.cpp:62, 75), so max_search_time_ = N makes its time cut end the search at loop iteration N + 1:
// the iteration cap of the device.  TEST INFRASTRUCTURE ONLY (hidden visibility: this ros::Time never meets
// ref_standin's).
#pragma once
#include <algorithm>
#include <cmath>
#include <iostream>
#include <limits>
#include <map>
#include <memory>
#include <string>
#include <vector>

#define ROS_ERROR(...) do {} while (0)
#define ROS_WARN(...) do {} while (0)
#define ROS_INFO(...) do {} while (0)
#define ROS_INFO_STREAM(x) do {} while (0)
#define ROS_WARN_THROTTLE(...) do {} while (0)

namespace ros {
struct Duration {
  double sec;
  double toSec() const { return sec; }
};
struct Time {
  double sec = 0.0;
  static double& clock() {
    static double t = 0.0;
    return t;
  }
  static Time now() {
    Time t;
    t.sec = clock();
    clock() += 1.0;
    return t;
  }
  Duration operator-(const Time& o) const { return Duration{ sec - o.sec }; }
};
inline bool ok() { return true; }
class NodeHandle {
public:
  std::map<std::string, double> values;
  template <typename T>
  bool param(const std::string& key, T& out, const T& def) const {
    auto it = values.find(key);
    if (it == values.end()) {
      out = def;
      return false;
    }
    out = static_cast<T>(it->second);
    return true;
  }
};
}  // namespace ros
