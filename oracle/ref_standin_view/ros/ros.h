// Stand-in for ros/ros.h in oracle/_ref/libfuel_ref_view.so: the tick clock of ../../ref_standin_astar/ros/ros.h for
// every translation unit of that library, so that Astar::search's time cut is the iteration cap there too, whichever
// other stand-in directory (ref_standin, for the Eigen that frontier_finder.cpp needs) comes next.  TEST INFRASTRUCTURE
// ONLY.
#pragma once
#include "../../ref_standin_astar/ros/ros.h"
