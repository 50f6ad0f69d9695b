# Build / test entry points. The reference's Makefile is a bare `nvcc -shared` of csrc/* into
# communicator.so with no arch flags; here every unit is compiled for sm_90a (H100) only
# (see adapcc_b200/build.py for the exact nvcc line).
PY ?= python

all: lib

lib:
	$(PY) -m adapcc_b200.build

force:
	$(PY) -m adapcc_b200.build --force --verbose

# the reference's name for the shared object, for scripts that dlopen ./communicator.so
communicator.so: lib
	cp adapcc_b200/_C/libadapcc.so communicator.so

test:
	$(PY) -m pytest tests -x -q -m "not gpu"

test-gpu:
	$(PY) -m pytest tests -x -q -m gpu

sass:
	$(PY) tools/sass_report.py

strategies:
	$(PY) tools/gen_strategies.py

clean:
	rm -rf adapcc_b200/_C communicator.so

.PHONY: all lib force test test-gpu sass strategies clean
