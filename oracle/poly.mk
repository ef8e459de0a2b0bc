# Builds the waypoint-polynomial oracle and, where the reference's sources are present, the reference's own
# poly_traj/src/polynomial_traj.cpp (compiled UNMODIFIED) with the driver ref_poly_wrap.cpp.  TEST INFRASTRUCTURE ONLY.
#   make -C oracle -f poly.mk     (oracle/poly.py: build())
# Flags as in the Makefile: -O3, no FMA contraction (the reference's Release build on x86-64 has none), and
# -fno-builtin-pow on both sides so that every pow() is libm's rather than whatever the compiler folds it into.
# The reference side compiles against ref_standin_poly/ alone (the Eigen pieces polynomial_traj.cpp uses; its inverse()
# is the oracle's orc_lu_inverse), with hidden visibility like _ref/libfuel_ref_traj.so.
CC := gcc
CFLAGS = -O3 -std=gnu11 -fPIC -ffp-contract=off -fno-builtin-pow -Wall -Wextra -Wno-unused-parameter

REFROOT := /root/reference/fuel_planner
REF_SRC := $(REFROOT)/poly_traj/src/polynomial_traj.cpp
REF_HDR := $(REFROOT)/poly_traj/include/poly_traj/polynomial_traj.h

ifneq ($(wildcard $(REF_SRC)),)
all: libfuel_oracle_poly.so _ref/libfuel_ref_poly.so
else
all: libfuel_oracle_poly.so
endif

libfuel_oracle_poly.so: fuel_oracle_poly.c fuel_oracle_poly.h
	$(CC) $(CFLAGS) -shared -o $@ fuel_oracle_poly.c -lm

_ref/libfuel_ref_poly.so: ref_poly_wrap.cpp $(wildcard ref_standin_poly/*/*) $(REF_SRC) $(REF_HDR) libfuel_oracle_poly.so
	mkdir -p _ref
	g++ -O3 -std=c++14 -fPIC -ffp-contract=off -fno-builtin-pow -w -shared -fvisibility=hidden \
	    -fvisibility-inlines-hidden -I ref_standin_poly -I $(REFROOT)/poly_traj/include -o $@ $(REF_SRC) \
	    ref_poly_wrap.cpp -L. -lfuel_oracle_poly -Wl,-rpath,'$$ORIGIN/..' -Wl,--no-undefined

clean:
	rm -f libfuel_oracle_poly.so _ref/libfuel_ref_poly.so
