# Builds, where the reference's sources are present, oracle/_ref/libfuel_ref_plan_yaw.so: the reference's own
# bspline/src/non_uniform_bspline.cpp (compiled UNMODIFIED) with the planYaw driver ref_plan_yaw_wrap.cpp, and the
# dim_ == 1, three-end-state combineCost driver ref_plan_yaw_cost_wrap.cpp over _ref/libfuel_ref.so's BsplineOptimizer.
# TEST INFRASTRUCTURE ONLY.
#   make -C oracle -f plan_yaw.mk      (oracle/plan_yaw.py: build(); needs _ref/libfuel_ref.so from the Makefile first)
# Flags as in the Makefile: -O3, no FMA contraction (the reference's Release build on x86-64 has none).
# The B-spline side compiles against ref_standin_traj/ first, then ref_standin/, with hidden visibility like
# _ref/libfuel_ref_traj.so; the optimizer driver compiles against ref_standin/ alone with default visibility, so that it
# shares libfuel_ref.so's optimizer code and NLopt stand-in recorder.
REFROOT := /root/reference/fuel_planner
REF_SRC := $(REFROOT)/bspline/src/non_uniform_bspline.cpp
HIDDEN := -fvisibility=hidden -fvisibility-inlines-hidden
CXX_REF := g++ -O3 -std=c++14 -fPIC -ffp-contract=off -w

ifneq ($(wildcard $(REF_SRC)),)
all: _ref/libfuel_ref_plan_yaw.so
else
all:
endif

_ref/plan_yaw_bspline.o: $(REF_SRC) $(wildcard ref_standin_traj/*/*) $(wildcard ref_standin/*) $(wildcard ref_standin/*/*)
	mkdir -p _ref
	$(CXX_REF) $(HIDDEN) -I ref_standin_traj -I ref_standin -I $(REFROOT)/plan_env/include -I $(REFROOT)/bspline/include \
	    -c -o $@ $(REF_SRC)

_ref/plan_yaw_wrap.o: ref_plan_yaw_wrap.cpp $(wildcard ref_standin_traj/*/*) $(wildcard ref_standin/*) $(wildcard ref_standin/*/*)
	mkdir -p _ref
	$(CXX_REF) $(HIDDEN) -I ref_standin_traj -I ref_standin -I $(REFROOT)/plan_env/include -I $(REFROOT)/bspline/include \
	    -c -o $@ ref_plan_yaw_wrap.cpp

_ref/plan_yaw_cost_wrap.o: ref_plan_yaw_cost_wrap.cpp $(wildcard ref_standin/*) $(wildcard ref_standin/*/*)
	mkdir -p _ref
	$(CXX_REF) -I ref_standin -I $(REFROOT)/plan_env/include -I $(REFROOT)/bspline_opt/include \
	    -I $(REFROOT)/active_perception/include -c -o $@ ref_plan_yaw_cost_wrap.cpp

_ref/libfuel_ref_plan_yaw.so: _ref/plan_yaw_bspline.o _ref/plan_yaw_wrap.o _ref/plan_yaw_cost_wrap.o _ref/libfuel_ref.so
	$(CXX_REF) -shared -o $@ _ref/plan_yaw_bspline.o _ref/plan_yaw_wrap.o _ref/plan_yaw_cost_wrap.o -L_ref -lfuel_ref \
	    -Wl,-rpath,'$$ORIGIN' -Wl,--no-undefined

clean:
	rm -f _ref/libfuel_ref_plan_yaw.so _ref/plan_yaw_bspline.o _ref/plan_yaw_wrap.o _ref/plan_yaw_cost_wrap.o
