# Builds the parameterization oracle and, where the reference's sources are present, the reference's own
# bspline/src/non_uniform_bspline.cpp (compiled UNMODIFIED) with the driver ref_param_wrap.cpp.  TEST INFRASTRUCTURE ONLY.
#   make -C oracle -f param.mk    (oracle/param.py: build(); needs libfuel_oracle.so and libfuel_oracle_traj.so first)
# Flags as in the Makefile: -O3, no FMA contraction (the reference's Release build on x86-64 has none).
# The reference side compiles against ref_standin_param/ first (the Eigen stand-in whose colPivHouseholderQr().solve()
# records the system and returns the oracle's orc_lstsq_colpiv_qr), then ref_standin_traj/ and ref_standin/, with
# hidden visibility like _ref/libfuel_ref_traj.so, so the two copies of the reference's code never bind to each other.
CC := gcc
CFLAGS = -O3 -std=gnu11 -fPIC -ffp-contract=off -Wall -Wextra -Wno-unused-parameter

REFROOT := /root/reference/fuel_planner
REF_SRC := $(REFROOT)/bspline/src/non_uniform_bspline.cpp

ifneq ($(wildcard $(REF_SRC)),)
all: libfuel_oracle_param.so _ref/libfuel_ref_param.so
else
all: libfuel_oracle_param.so
endif

libfuel_oracle_param.so: fuel_oracle_param.c fuel_oracle_param.h fuel_oracle_traj.h fuel_oracle.h libfuel_oracle.so \
                         libfuel_oracle_traj.so
	$(CC) $(CFLAGS) -shared -o $@ fuel_oracle_param.c -L. -lfuel_oracle_traj -lfuel_oracle -Wl,-rpath,'$$ORIGIN' -lm

_ref/libfuel_ref_param.so: ref_param_wrap.cpp $(wildcard ref_standin_param/*/*) $(wildcard ref_standin_traj/*/*) \
                           $(wildcard ref_standin/*) $(wildcard ref_standin/*/*) $(REF_SRC) libfuel_oracle_param.so
	mkdir -p _ref
	g++ -O3 -std=c++14 -fPIC -ffp-contract=off -w -shared -fvisibility=hidden -fvisibility-inlines-hidden \
	    -I ref_standin_param -I ref_standin_traj -I ref_standin -I $(REFROOT)/plan_env/include \
	    -I $(REFROOT)/bspline/include -o $@ $(REF_SRC) ref_param_wrap.cpp \
	    -L. -lfuel_oracle_param -Wl,-rpath,'$$ORIGIN/..' -Wl,--no-undefined

clean:
	rm -f libfuel_oracle_param.so _ref/libfuel_ref_param.so
