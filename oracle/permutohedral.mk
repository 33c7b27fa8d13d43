# Builds oracle/_ref/libpermutohedral_ref.so (test infrastructure): the reference's UNMODIFIED
# third_party/permutohedral/permutohedral.cpp, compiled as its setup.py compiles the probreg._permutohedral_lattice extension
# (setuptools' default optimisation, -std=c++14, -fvisibility=hidden, no -march: SSE2 but not SSE4.1, so the SSE lattice build with
# _mm_cvtps_epi32 rounding), against this directory's Eigen/Core shim and C entry point.
#   make -f oracle/permutohedral.mk REF=<reference checkout>
HERE := $(abspath $(dir $(lastword $(MAKEFILE_LIST))))
REF ?= $(PROBREG_REFERENCE)
CXX ?= g++
OUT := $(HERE)/_ref/libpermutohedral_ref.so
SRC := $(REF)/third_party/permutohedral/permutohedral.cpp
ifneq ($(shell uname -m),x86_64)
$(error the reference lattice oracle needs an x86-64 host: elsewhere permutohedral.cpp compiles its non-SSE path, which rounds differently)
endif
ifeq ($(REF),)
$(error REF (or PROBREG_REFERENCE) must name a checkout of the reference)
endif

$(OUT): $(SRC) $(HERE)/permutohedral/ref_capi.cpp $(HERE)/permutohedral/Eigen/Core
	mkdir -p $(HERE)/_ref
	$(CXX) -O3 -DNDEBUG -fwrapv -fPIC -shared -std=c++14 -fvisibility=hidden -I$(HERE)/permutohedral -I$(REF)/third_party/permutohedral \
	    -o $@ $(SRC) $(HERE)/permutohedral/ref_capi.cpp
