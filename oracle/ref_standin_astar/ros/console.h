// Stand-in for ros/console.h: the log macros of ros.h in this directory.  TEST INFRASTRUCTURE ONLY.
#pragma once
#include "ros.h"
