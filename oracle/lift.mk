# Builds libliftoracle.so: the restated hash-to-curve and initial global cumulative sum (lift.hpp, lift_capi.cpp) for the tests of
# sp1b200_program_vk_tail.  Header-only over core.hpp and poseidon2.hpp, so it links nothing else.  Test infrastructure only; never linked
# into the product library.
#   make -C oracle -f lift.mk
CXX := /usr/bin/g++
CXXFLAGS ?= -O3 -march=x86-64-v3 -std=c++17 -fPIC -fopenmp -Wall -Wextra -Wno-unused-function
HDRS := field.hpp core.hpp poseidon2.hpp poseidon2_rc.inc lift.hpp

all: libliftoracle.so

libliftoracle.so: lift_capi.cpp $(HDRS) lift.mk
	$(CXX) $(CXXFLAGS) -shared -o $@.tmp lift_capi.cpp
	mv -f $@.tmp $@

clean:
	rm -f libliftoracle.so
.PHONY: all clean
