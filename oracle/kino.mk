# Builds the kinodynamic-search oracle: kinodynamicReplan's search, retry and getSamples restated in C
# (fuel_oracle_kino.c), with the host build of the device's math header (kino_math_host.cpp); and, where the reference's
# sources are present, oracle/_ref/libfuel_ref_kino.so: the reference's own path_searching/src/kinodynamic_astar.cpp
# (compiled UNMODIFIED) with the driver ref_kino_wrap.cpp, over the SDFMap of _ref/libfuel_ref.so.
# TEST INFRASTRUCTURE ONLY.
#   make -C oracle -f kino.mk    (oracle/kino.py: build(); the reference part needs _ref/libfuel_ref.so first)
# -O3 without FMA contraction, like the reference's Release build on x86-64; libquadmath (part of gcc) gives the
# correctly rounded acos / cos of the oracle's DEVICE mode.  The reference side compiles against ref_standin_kino/
# first (the Eigen pieces kinodynamic_astar.cpp uses), then ref_standin_astar/ (ros/console.h, boost's hash header),
# then ref_standin/, with hidden visibility like _ref/libfuel_ref_astar.so.
CC := gcc
CXX := g++
CFLAGS = -O3 -std=gnu11 -fPIC -ffp-contract=off -Wall -Wextra -Wno-unused-parameter
CXXFLAGS = -O3 -std=c++14 -fPIC -ffp-contract=off -Wall -Wextra -I ../fuel_b200/csrc

REFROOT := /root/reference/fuel_planner
REF_SRC := $(REFROOT)/path_searching/src/kinodynamic_astar.cpp
HIDDEN := -fvisibility=hidden -fvisibility-inlines-hidden
CXX_REF := g++ -O3 -std=c++14 -fPIC -ffp-contract=off -w

ifneq ($(wildcard $(REF_SRC)),)
all: libfuel_oracle_kino.so _ref/libfuel_ref_kino.so
else
all: libfuel_oracle_kino.so
endif

libfuel_oracle_kino.so: fuel_oracle_kino.c fuel_oracle_kino.h fuel_oracle_astar.h kino_math_host.cpp ../fuel_b200/csrc/kino_math.cuh
	$(CC) $(CFLAGS) -c -o fuel_oracle_kino.o fuel_oracle_kino.c
	$(CXX) $(CXXFLAGS) -c -o kino_math_host.o kino_math_host.cpp
	$(CXX) -shared -o $@ fuel_oracle_kino.o kino_math_host.o -lquadmath -lm
	rm -f fuel_oracle_kino.o kino_math_host.o

_ref/libfuel_ref_kino.so: ref_kino_wrap.cpp $(REF_SRC) $(wildcard ref_standin_kino/*/*) $(wildcard ref_standin_astar/*/*) \
                          $(wildcard ref_standin_astar/*/*/*) $(wildcard ref_standin/*/*) _ref/libfuel_ref.so
	mkdir -p _ref
	$(CXX_REF) $(HIDDEN) -shared -I ref_standin_kino -I ref_standin_astar -I ref_standin -I $(REFROOT)/plan_env/include \
	    -I $(REFROOT)/path_searching/include -o $@ $(REF_SRC) ref_kino_wrap.cpp -L_ref -lfuel_ref \
	    -Wl,-rpath,'$$ORIGIN' -Wl,--no-undefined

clean:
	rm -f libfuel_oracle_kino.so _ref/libfuel_ref_kino.so
