# Builds the A* oracle and, where the reference's sources are present, oracle/_ref/libfuel_ref_astar.so: the reference's
# own path_searching/src/astar2.cpp (compiled UNMODIFIED) with the driver ref_astar_wrap.cpp, over the SDFMap and
# RayCaster of _ref/libfuel_ref.so.  TEST INFRASTRUCTURE ONLY.
#   make -C oracle -f astar.mk    (oracle/astar.py: build(); needs _ref/libfuel_ref.so from the Makefile first)
# Flags as in the Makefile: -O3, no FMA contraction (the reference's Release build on x86-64 has none).  The reference
# side compiles against ref_standin_astar/ first (the Eigen pieces astar2.cpp uses, ros/console.h, boost's hash header,
# the tick clock), then ref_standin/, with hidden visibility like _ref/libfuel_ref_traj.so, so that its ros::Time and
# inline functions never bind to the ones of _ref/libfuel_ref.so.
CC := gcc
CFLAGS = -O3 -std=gnu11 -fPIC -ffp-contract=off -Wall -Wextra -Wno-unused-parameter

REFROOT := /root/reference/fuel_planner
REF_SRC := $(REFROOT)/path_searching/src/astar2.cpp
HIDDEN := -fvisibility=hidden -fvisibility-inlines-hidden
CXX_REF := g++ -O3 -std=c++14 -fPIC -ffp-contract=off -w

ifneq ($(wildcard $(REF_SRC)),)
all: libfuel_oracle_astar.so _ref/libfuel_ref_astar.so
else
all: libfuel_oracle_astar.so
endif

libfuel_oracle_astar.so: fuel_oracle_astar.c fuel_oracle_astar.h
	$(CC) $(CFLAGS) -shared -o $@ fuel_oracle_astar.c -lm

_ref/libfuel_ref_astar.so: ref_astar_wrap.cpp $(REF_SRC) $(wildcard ref_standin_astar/*/*) $(wildcard ref_standin_astar/*/*/*) \
                           $(wildcard ref_standin/*/*) _ref/libfuel_ref.so
	mkdir -p _ref
	$(CXX_REF) $(HIDDEN) -shared -I ref_standin_astar -I ref_standin -I $(REFROOT)/plan_env/include \
	    -I $(REFROOT)/path_searching/include -o $@ $(REF_SRC) ref_astar_wrap.cpp -L_ref -lfuel_ref \
	    -Wl,-rpath,'$$ORIGIN' -Wl,--no-undefined

clean:
	rm -f libfuel_oracle_astar.so _ref/libfuel_ref_astar.so
