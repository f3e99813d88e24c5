# Builds oracle/_ref/libsp1ref_lift.so: the reference's hash-to-curve primitives (sp1-gpu/crates/sys/include/fields/
# kb31_septic_extension_t.cuh and poseidon2/poseidon2.cuh, compiled unmodified from where they lie) behind oracle/ref_lift.cu, for
# tests/test_ref_lift.py.
# Built only where /root/reference exists; elsewhere the prebuilt library (oracle/_ref/ is git-ignored) is used if present.
#   make -C oracle -f ref_lift.mk
REF := /root/reference/sp1-gpu/crates/sys
NVCC ?= /usr/local/cuda/bin/nvcc
FLAGS := -gencode arch=compute_90a,code=sm_90a -std=c++20 -O3 --expt-relaxed-constexpr -Xcompiler -fPIC -DFEATURE_KOALA_BEAR \
	-I$(REF)/include -ccbin /usr/bin/g++ -w

ifneq ($(wildcard $(REF)/include/fields/kb31_septic_extension_t.cuh),)
all: _ref/libsp1ref_lift.so
else
all:
	@test -f _ref/libsp1ref_lift.so && echo "oracle/_ref: using the prebuilt libsp1ref_lift.so (/root/reference absent)" || echo "oracle/_ref: libsp1ref_lift.so unavailable (/root/reference absent, nothing prebuilt)"
endif

_ref/libsp1ref_lift.so: ref_lift.cu ref_lift.mk
	@mkdir -p _ref
	$(NVCC) $(FLAGS) -shared -o $@.tmp $< -lcudart
	mv -f $@.tmp $@

.PHONY: all
