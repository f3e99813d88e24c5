# convenience targets; the driver uses __graft_entry__.py, pytest and bench.py directly
PY ?= python
.PHONY: build test test-gpu bench bench-ref smoke golden clean
build:
	$(PY) __graft_entry__.py
test: build
	$(PY) -m pytest tests -q -m "not gpu"
test-gpu: build
	$(PY) -m pytest tests -q -m gpu
smoke: build
	$(PY) __graft_entry__.py smoke
bench:
	$(PY) bench.py
bench-ref:
	$(PY) bench.py --impl reference
golden:
	$(PY) tools/gen_golden_proofs.py
clean:
	$(MAKE) -C sp1_b200/csrc clean
	$(MAKE) -C examples clean
	rm -f oracle/liboracle.so oracle/libdebugoracle.so
