# Builds the global-tour oracle: fuel_oracle_gtour.c (Held-Karp over findGlobalTour's integer ATSP) into
# libfuel_oracle_gtour.so, and, where the reference's sources are present, oracle/_ref/libfuel_ref_gtour.so: the
# reference's fast_exploration_manager.cpp (findGlobalTour), frontier_finder.cpp, graph_node.cpp, perception_utils.cpp
# and astar2.cpp, each UNMODIFIED and compiled as tour.mk compiles them, with the real LKH (utils/lkh_tsp_solver: its
# src/*.c and lkh_interface.cpp) in place of tour.mk's stub of solveTSPLKH, and the driver ref_gtour_wrap.cpp, over the
# SDFMap and RayCaster of _ref/libfuel_ref.so.  TEST INFRASTRUCTURE ONLY.
#   make -C oracle -f gtour.mk    (oracle/gtour.py: build(); needs _ref/libfuel_ref.so from the Makefile first)
# LKH's headers define its globals without extern, so its C files need -fcommon; only lkh_interface.cpp includes LKH.h
# (the other files see ref_standin_tour's declaration of solveTSPLKH alone).  Hidden visibility keeps LKH's globals
# (c, C, D, ...) and this library's ViewNode statics, FrontierFinder, Astar and ros::Time apart from the other
# reference libraries'.
CC := gcc
CFLAGS = -O3 -std=gnu11 -fPIC -ffp-contract=off -Wall -Wextra -Wno-unused-parameter

REFROOT := /root/reference/fuel_planner
AP := $(REFROOT)/active_perception
EM := $(REFROOT)/exploration_manager
LKH := $(REFROOT)/utils/lkh_tsp_solver
ASTAR_SRC := $(REFROOT)/path_searching/src/astar2.cpp
TOUR_SRC := $(EM)/src/fast_exploration_manager.cpp $(AP)/src/graph_node.cpp $(AP)/src/frontier_finder.cpp \
            $(AP)/src/perception_utils.cpp
LKH_C := $(wildcard $(LKH)/src/*.c)
HIDDEN := -fvisibility=hidden -fvisibility-inlines-hidden
CXX_REF := g++ -O3 -std=c++14 -fPIC -ffp-contract=off -w
TOUR_INC := -I ref_standin_tour -I ref_standin_view -I $(AP)/include -I ref_standin -I ref_standin_astar \
            -I $(REFROOT)/plan_env/include -I $(REFROOT)/path_searching/include -I $(EM)/include

ifneq ($(wildcard $(LKH)/src/lkh_interface.cpp),)
all: libfuel_oracle_gtour.so _ref/libfuel_ref_gtour.so
else
all: libfuel_oracle_gtour.so
endif

libfuel_oracle_gtour.so: fuel_oracle_gtour.c fuel_oracle_gtour.h
	$(CC) $(CFLAGS) -shared -o $@ fuel_oracle_gtour.c

_ref/libfuel_ref_gtour.so: ref_gtour_wrap.cpp $(TOUR_SRC) $(ASTAR_SRC) $(LKH_C) $(LKH)/src/lkh_interface.cpp \
                           $(wildcard ref_standin_tour/*/*) $(wildcard ref_standin_view/*/*) \
                           $(wildcard ref_standin_astar/*/*) $(wildcard ref_standin_astar/*/*/*) \
                           $(wildcard ref_standin/*/*) $(wildcard ref_standin/*/*/*) _ref/libfuel_ref.so
	mkdir -p _ref/gtour_obj/lkh
	for f in $(LKH_C); do \
	    gcc -O3 -fPIC -fcommon $(HIDDEN) -w -I $(LKH)/include -c $$f -o _ref/gtour_obj/lkh/$$(basename $$f .c).o \
	    || exit 1; done
	$(CXX_REF) $(HIDDEN) -fcommon -I $(LKH)/include -c $(LKH)/src/lkh_interface.cpp -o _ref/gtour_obj/lkh_interface.o
	$(CXX_REF) $(HIDDEN) -I ref_standin_view -I ref_standin_astar -I ref_standin \
	    -I $(REFROOT)/plan_env/include -I $(REFROOT)/path_searching/include -c $(ASTAR_SRC) -o _ref/gtour_obj/astar2.o
	for f in $(TOUR_SRC) ref_gtour_wrap.cpp; do \
	    $(CXX_REF) $(HIDDEN) $(TOUR_INC) -c $$f -o _ref/gtour_obj/$$(basename $$f .cpp).o || exit 1; done
	$(CXX_REF) -shared -o $@ _ref/gtour_obj/*.o _ref/gtour_obj/lkh/*.o -L_ref -lfuel_ref -L. -lfuel_oracle -lm \
	    -Wl,-rpath,'$$ORIGIN' -Wl,-rpath,'$$ORIGIN/..' -Wl,--no-undefined

clean:
	rm -rf libfuel_oracle_gtour.so _ref/libfuel_ref_gtour.so _ref/gtour_obj
