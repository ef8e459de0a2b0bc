// Stand-in for the bspline/Bspline message that exploration_manager/expl_data.h names in FSMData.  TEST
// INFRASTRUCTURE ONLY.
#pragma once
namespace bspline {
struct Bspline {};
}  // namespace bspline
