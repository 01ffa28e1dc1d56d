# Repo-level developer targets (the reference's root Makefile renders the cookiecutter template as its only "test").
PY ?= python

help:
	@echo "make build          compile the native module for sm_90a (nvcc) and import the package"
	@echo "make test           CPU test-suite (gloo, 2 ranks)"
	@echo "make test-gpu       GPU test-suite (needs an H100)"
	@echo "make template-test  render a project skeleton into /tmp and list it (reference: cookiecutter --no-input)"
	@echo "make bench          headline benchmark JSON line (1 GPU)"
	@echo "make clean          remove build artefacts"

build:
	$(PY) __graft_entry__.py

test:
	$(PY) -m pytest tests -x -q -m "not gpu"

test-gpu:
	$(PY) -m pytest tests -x -q -m gpu

template-test:
	rm -rf /tmp/ddl_template_test && $(PY) -m distributeddeeplearning_b200.cli new-project --name mstestdist --path /tmp/ddl_template_test \
		&& find /tmp/ddl_template_test -type f | sort

bench:
	$(PY) bench.py --gpus 1 --steps 30 --warmup 5

clean:
	rm -rf distributeddeeplearning_b200/csrc/build distributeddeeplearning_b200/_C.so /tmp/ddl_template_test

.PHONY: help build test test-gpu template-test bench clean
