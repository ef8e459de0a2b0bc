# Builds the trajectory-check oracle and, where the reference's sources are present, the reference's own
# bspline/src/non_uniform_bspline.cpp (compiled UNMODIFIED) with its test driver.  TEST INFRASTRUCTURE ONLY.
#   make -C oracle -f traj.mk     (oracle/traj.py: build(); needs libfuel_oracle.so from the Makefile first)
# Flags as in the Makefile: -O3, no FMA contraction (the reference's Release build on x86-64 has none).
# The reference side compiles against ref_standin_traj/ first (VectorXd and the other Eigen pieces the B-spline class
# uses, ROS_ERROR_COND; each file says what it stands for), then ref_standin/.  Hidden visibility keeps the stand-in's
# inline functions from binding to those of _ref/libfuel_ref.so, whose SDFMap objects the driver reads.
CC := gcc
CFLAGS = -O3 -std=gnu11 -fPIC -ffp-contract=off -Wall -Wextra -Wno-unused-parameter

REFROOT := /root/reference/fuel_planner
REF_SRC := $(REFROOT)/bspline/src/non_uniform_bspline.cpp

ifneq ($(wildcard $(REF_SRC)),)
all: libfuel_oracle_traj.so _ref/libfuel_ref_traj.so
else
all: libfuel_oracle_traj.so
endif

libfuel_oracle_traj.so: fuel_oracle_traj.c fuel_oracle_traj.h fuel_oracle.h libfuel_oracle.so
	$(CC) $(CFLAGS) -shared -o $@ fuel_oracle_traj.c -L. -lfuel_oracle -Wl,-rpath,'$$ORIGIN' -lm

_ref/libfuel_ref_traj.so: ref_traj_wrap.cpp $(wildcard ref_standin_traj/*/*) $(wildcard ref_standin/*) \
                          $(wildcard ref_standin/*/*) $(REF_SRC)
	mkdir -p _ref
	g++ -O3 -std=c++14 -fPIC -ffp-contract=off -w -shared -fvisibility=hidden -fvisibility-inlines-hidden \
	    -I ref_standin_traj -I ref_standin -I $(REFROOT)/plan_env/include -I $(REFROOT)/bspline/include \
	    -o $@ $(REF_SRC) ref_traj_wrap.cpp -Wl,--no-undefined

clean:
	rm -f libfuel_oracle_traj.so _ref/libfuel_ref_traj.so
