# Builds oracle/_ref/libsp1ref_septic.so: the reference's septic-curve arithmetic (sp1-gpu/crates/sys/include/fields/
# kb31_septic_extension_t.cuh, compiled unmodified from where it lies) behind oracle/ref_septic.cu, for tests/test_ref_septic.py.
# Built only where /root/reference exists; elsewhere the prebuilt library (oracle/_ref/ is git-ignored) is used if present.
#   make -C oracle -f ref_septic.mk
REF := /root/reference/sp1-gpu/crates/sys
NVCC ?= /usr/local/cuda/bin/nvcc
FLAGS := -gencode arch=compute_90a,code=sm_90a -std=c++20 -O3 --expt-relaxed-constexpr -Xcompiler -fPIC -DFEATURE_KOALA_BEAR \
	-I$(REF)/include -ccbin /usr/bin/g++ -w

ifneq ($(wildcard $(REF)/include/fields/kb31_septic_extension_t.cuh),)
all: _ref/libsp1ref_septic.so
else
all:
	@test -f _ref/libsp1ref_septic.so && echo "oracle/_ref: using the prebuilt libsp1ref_septic.so (/root/reference absent)" || echo "oracle/_ref: libsp1ref_septic.so unavailable (/root/reference absent, nothing prebuilt)"
endif

_ref/libsp1ref_septic.so: ref_septic.cu ref_septic.mk
	@mkdir -p _ref
	$(NVCC) $(FLAGS) -shared -o $@.tmp $< -lcudart
	mv -f $@.tmp $@

.PHONY: all
