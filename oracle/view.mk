# Builds the view-cost oracle (fuel_oracle_view.c over the A* oracle fuel_oracle_astar.c, both compiled into
# libfuel_oracle_view.so) and, where the reference's sources are present, oracle/_ref/libfuel_ref_view.so: the
# reference's graph_node.cpp (ViewNode::searchPath / computeCost) and frontier_finder.cpp + perception_utils.cpp (the cost
# bookkeeping), each UNMODIFIED, with their own copy of astar2.cpp and the driver ref_view_wrap.cpp, over the SDFMap and
# RayCaster of _ref/libfuel_ref.so.  TEST INFRASTRUCTURE ONLY.
#   make -C oracle -f view.mk    (oracle/view.py: build(); needs _ref/libfuel_ref.so from the Makefile first)
# Flags as in astar.mk: -O3, no FMA contraction.  Every reference unit sees the tick clock first
# (ref_standin_view/ros/ros.h).  astar2.cpp takes its Eigen from ref_standin_astar; the others take ref_standin's
# (frontier_finder.cpp needs its matrices) and the REAL active_perception headers ahead of ref_standin's graph_node.h
# stand-in, which only libfuel_ref.so uses.  Both Eigen stand-ins define the same Vec3 layout.  Hidden visibility keeps
# this library's FrontierFinder, Astar and ros::Time apart from libfuel_ref.so's.
CC := gcc
CFLAGS = -O3 -std=gnu11 -fPIC -ffp-contract=off -Wall -Wextra -Wno-unused-parameter

REFROOT := /root/reference/fuel_planner
AP := $(REFROOT)/active_perception
ASTAR_SRC := $(REFROOT)/path_searching/src/astar2.cpp
VIEW_SRC := $(AP)/src/graph_node.cpp $(AP)/src/frontier_finder.cpp $(AP)/src/perception_utils.cpp
HIDDEN := -fvisibility=hidden -fvisibility-inlines-hidden
CXX_REF := g++ -O3 -std=c++14 -fPIC -ffp-contract=off -w
VIEW_INC := -I ref_standin_view -I $(AP)/include -I ref_standin -I ref_standin_astar -I $(REFROOT)/plan_env/include \
            -I $(REFROOT)/path_searching/include

ifneq ($(wildcard $(AP)/src/graph_node.cpp),)
all: libfuel_oracle_view.so _ref/libfuel_ref_view.so
else
all: libfuel_oracle_view.so
endif

libfuel_oracle_view.so: fuel_oracle_view.c fuel_oracle_view.h fuel_oracle_astar.c fuel_oracle_astar.h
	$(CC) $(CFLAGS) -shared -o $@ fuel_oracle_view.c fuel_oracle_astar.c -lm

_ref/libfuel_ref_view.so: ref_view_wrap.cpp $(VIEW_SRC) $(ASTAR_SRC) $(wildcard ref_standin_view/*/*) \
                          $(wildcard ref_standin_astar/*/*) $(wildcard ref_standin_astar/*/*/*) $(wildcard ref_standin/*/*) \
                          $(wildcard ref_standin/*/*/*) _ref/libfuel_ref.so
	mkdir -p _ref/view_obj
	$(CXX_REF) $(HIDDEN) -I ref_standin_view -I ref_standin_astar -I ref_standin -I $(REFROOT)/plan_env/include \
	    -I $(REFROOT)/path_searching/include -c $(ASTAR_SRC) -o _ref/view_obj/astar2.o
	for f in $(VIEW_SRC) ref_view_wrap.cpp; do \
	    $(CXX_REF) $(HIDDEN) $(VIEW_INC) -c $$f -o _ref/view_obj/$$(basename $$f .cpp).o || exit 1; done
	$(CXX_REF) -shared -o $@ _ref/view_obj/*.o -L_ref -lfuel_ref -L. -lfuel_oracle -Wl,-rpath,'$$ORIGIN' \
	    -Wl,-rpath,'$$ORIGIN/..' -Wl,--no-undefined

clean:
	rm -rf libfuel_oracle_view.so _ref/libfuel_ref_view.so _ref/view_obj
