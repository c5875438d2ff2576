# convenience targets over __graft_entry__.build(), pytest and bench.py
PY ?= python

build:            ## nvcc (sm_90a) -> csrc/libmm_engine.so, gcc -> oracle/liborc.so
	$(PY) -c "import __graft_entry__ as g; g.build()"

test:             ## CPU suite: oracle KATs / properties, golden fixtures, ABI export, host mirror, gloo sharding
	$(PY) -m pytest tests -x -q -m "not gpu"

test-gpu:         ## parity through the C ABI (needs an H100)
	$(PY) -m pytest tests -x -q -m gpu

smoke:            ## one small tick on cuda:0, checked against the oracle
	$(PY) __graft_entry__.py --smoke

bench:            ## the contract line (N = 1); `make bench-ref` = CPU restatement on all host cores
	$(PY) bench.py
bench-ref:
	$(PY) bench.py --impl reference

.PHONY: build test test-gpu smoke bench bench-ref
