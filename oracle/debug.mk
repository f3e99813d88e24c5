# Builds libdebugoracle.so: the restated shard checks (debug.hpp, debug_capi.cpp) for the tests of sp1b200_debug_constraints /
# sp1b200_debug_interactions.  Test infrastructure only; never linked into the product library.
#   make -C oracle -f debug.mk
CXX := /usr/bin/g++
CXXFLAGS ?= -O3 -march=x86-64-v3 -std=c++17 -fPIC -fopenmp -Wall -Wextra -Wno-unused-function
HDRS := $(wildcard *.hpp) poseidon2_rc.inc

all: libdebugoracle.so

libdebugoracle.so: debug_capi.cpp $(HDRS) debug.mk
	$(CXX) $(CXXFLAGS) -shared -o $@.tmp debug_capi.cpp
	mv -f $@.tmp $@

clean:
	rm -f libdebugoracle.so
.PHONY: all clean
