// Stand-in for utils/lkh_tsp_solver/include/lkh_tsp_solver/lkh_interface.h: the one function
// fast_exploration_manager.cpp calls (the driver oracle/ref_tour_wrap.cpp defines it; the local tour never reaches it).
// TEST INFRASTRUCTURE ONLY.
#pragma once
int solveTSPLKH(const char* input_file);
