// Stand-in for visualization_msgs/Marker.h: fast_exploration_manager.cpp includes it and uses nothing of it.  TEST
// INFRASTRUCTURE ONLY.
#pragma once
