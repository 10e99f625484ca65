# Convenience targets; everything also works without make (see README.md).
PY ?= python
.PHONY: build test test-gpu bench bench-ref smoke clean
build:            ## nvcc (sm_90a) -> litegs_b200/liblitegs_b200.so, gcc -> oracle/liborc.so, reference extensions + staged reference Python -> oracle/_ref (if a LiteGS checkout is found: $LITEGS_REFERENCE, ../reference, ../LiteGS)
	$(PY) -c "import __graft_entry__ as g; g.build()"
test:             ## CPU suite: oracle, golden vectors, ABI, gloo, data formats
	$(PY) -m pytest tests -q -m "not gpu"
test-gpu:         ## on an H100: parity tests through the C ABI
	$(PY) -m pytest tests -q -m gpu
smoke:
	$(PY) -c "import __graft_entry__ as g; g.smoke()"
bench:            ## one JSON line (N=1); N>1: python -m torch.distributed.run --nproc-per-node N bench.py --gpus N
	$(PY) bench.py
bench-ref:        ## the CPU arm
	$(PY) bench.py --impl reference
clean:
	rm -rf litegs_b200/_obj litegs_b200/liblitegs_b200.so oracle/liborc.so
