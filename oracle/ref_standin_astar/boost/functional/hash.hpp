// Stand-in for boost/functional/hash.hpp: astar2.h includes it, but its hash is matrix_hash.h's (std::hash per element).
// TEST INFRASTRUCTURE ONLY.
#pragma once
#include <functional>
