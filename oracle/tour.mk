# Builds the local-tour oracle: fuel_oracle_tour.c (refineLocalTour) over the view-cost and A* oracles, compiled into
# libfuel_oracle_tour.so, and, where the reference's sources are present, oracle/_ref/libfuel_ref_tour.so: the
# reference's fast_exploration_manager.cpp (refineLocalTour), graph_node.cpp, frontier_finder.cpp and
# perception_utils.cpp, each UNMODIFIED, with their own copy of astar2.cpp and the driver ref_tour_wrap.cpp, over the
# SDFMap and RayCaster of _ref/libfuel_ref.so.  TEST INFRASTRUCTURE ONLY.
#   make -C oracle -f tour.mk    (oracle/tour.py: build(); needs _ref/libfuel_ref.so from the Makefile first)
# Flags as in view.mk: -O3, no FMA contraction.  astar2.cpp is compiled as view.mk compiles it (ref_standin_astar's
# Eigen); the others take view.mk's include order with ref_standin_tour first: the
# planner manager, LKH, message and ROS stand-ins fast_exploration_manager.cpp needs (ros.h adds to ref_standin_view's
# tick clock, Eigen adds Quaterniond to ref_standin's).  Hidden visibility keeps this library's ViewNode statics,
# FrontierFinder, Astar and ros::Time apart from the other reference libraries'.
CC := gcc
CFLAGS = -O3 -std=gnu11 -fPIC -ffp-contract=off -Wall -Wextra -Wno-unused-parameter

REFROOT := /root/reference/fuel_planner
AP := $(REFROOT)/active_perception
EM := $(REFROOT)/exploration_manager
ASTAR_SRC := $(REFROOT)/path_searching/src/astar2.cpp
TOUR_SRC := $(EM)/src/fast_exploration_manager.cpp $(AP)/src/graph_node.cpp $(AP)/src/frontier_finder.cpp \
            $(AP)/src/perception_utils.cpp
HIDDEN := -fvisibility=hidden -fvisibility-inlines-hidden
CXX_REF := g++ -O3 -std=c++14 -fPIC -ffp-contract=off -w
TOUR_INC := -I ref_standin_tour -I ref_standin_view -I $(AP)/include -I ref_standin -I ref_standin_astar \
            -I $(REFROOT)/plan_env/include -I $(REFROOT)/path_searching/include -I $(EM)/include

ifneq ($(wildcard $(EM)/src/fast_exploration_manager.cpp),)
all: libfuel_oracle_tour.so _ref/libfuel_ref_tour.so
else
all: libfuel_oracle_tour.so
endif

libfuel_oracle_tour.so: fuel_oracle_tour.c fuel_oracle_tour.h fuel_oracle_view.c fuel_oracle_view.h \
                        fuel_oracle_astar.c fuel_oracle_astar.h
	$(CC) $(CFLAGS) -shared -o $@ fuel_oracle_tour.c fuel_oracle_view.c fuel_oracle_astar.c -lm

_ref/libfuel_ref_tour.so: ref_tour_wrap.cpp $(TOUR_SRC) $(ASTAR_SRC) $(wildcard ref_standin_tour/*/*) \
                          $(wildcard ref_standin_view/*/*) $(wildcard ref_standin_astar/*/*) \
                          $(wildcard ref_standin_astar/*/*/*) $(wildcard ref_standin/*/*) $(wildcard ref_standin/*/*/*) \
                          _ref/libfuel_ref.so
	mkdir -p _ref/tour_obj
	$(CXX_REF) $(HIDDEN) -I ref_standin_view -I ref_standin_astar -I ref_standin \
	    -I $(REFROOT)/plan_env/include -I $(REFROOT)/path_searching/include -c $(ASTAR_SRC) -o _ref/tour_obj/astar2.o
	for f in $(TOUR_SRC) ref_tour_wrap.cpp; do \
	    $(CXX_REF) $(HIDDEN) $(TOUR_INC) -c $$f -o _ref/tour_obj/$$(basename $$f .cpp).o || exit 1; done
	$(CXX_REF) -shared -o $@ _ref/tour_obj/*.o -L_ref -lfuel_ref -L. -lfuel_oracle -Wl,-rpath,'$$ORIGIN' \
	    -Wl,-rpath,'$$ORIGIN/..' -Wl,--no-undefined

clean:
	rm -rf libfuel_oracle_tour.so _ref/libfuel_ref_tour.so _ref/tour_obj
