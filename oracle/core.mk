# Builds libcoreoracle.so: the restated core-proof verifier (core.hpp, core_capi.cpp) for the tests of sp1b200_verify_core_proof.  It
# links liboracle.so (the restated ShardVerifier, oracle/Makefile) from the same directory.  Test infrastructure only; never linked
# into the product library.
#   make -C oracle -f core.mk
CXX := /usr/bin/g++
CXXFLAGS ?= -O3 -march=x86-64-v3 -std=c++17 -fPIC -fopenmp -Wall -Wextra -Wno-unused-function
HDRS := field.hpp core.hpp

all: libcoreoracle.so

libcoreoracle.so: core_capi.cpp $(HDRS) core.mk liboracle.so
	$(CXX) $(CXXFLAGS) -shared -o $@.tmp core_capi.cpp -L. -loracle -Wl,-rpath,'$$ORIGIN'
	mv -f $@.tmp $@

liboracle.so:
	$(MAKE) -f Makefile liboracle.so

clean:
	rm -f libcoreoracle.so
.PHONY: all clean
