// Stand-in for ros/ros.h as bspline/src/non_uniform_bspline.cpp uses it: the facilities of ../../ref_standin/ros/ros.h
// plus ROS_ERROR_COND (checkRatio's log line), which prints nothing.  TEST INFRASTRUCTURE ONLY.
#pragma once
#include "../../ref_standin/ros/ros.h"

#define ROS_ERROR_COND(...) do {} while (0)
