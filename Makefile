# Build / test entry points (reference counterpart: Makefile of NVIDIA-Merlin/distributed-embeddings)
PYTHON ?= python

all: build

build:
	$(PYTHON) -m distributed_embeddings_b200.ops._build

rebuild:
	$(PYTHON) -m distributed_embeddings_b200.ops._build --force -v

test:
	$(PYTHON) -m pytest tests -q -m "not gpu"

test-gpu:
	$(PYTHON) -m pytest tests -q -m gpu

# race / memory checks of the single-GPU kernels (run on a GPU box)
sanitize:
	compute-sanitizer --tool memcheck $(PYTHON) -m pytest tests/test_embedding_ops.py tests/test_dense_kernels.py -q -m gpu -x
	compute-sanitizer --tool racecheck $(PYTHON) -m pytest tests/test_dense_kernels.py -q -m gpu -x -k interaction

sass:
	$(PYTHON) tools/dump_sass.py
	$(PYTHON) tools/sass_census.py
	$(PYTHON) tools/resource_usage.py

bench:
	$(PYTHON) bench.py --gpus 1 --steps 50 --warmup 10

wheel: build
	$(PYTHON) setup.py -q bdist_wheel -d dist

clean:
	rm -rf distributed_embeddings_b200/_C.so distributed_embeddings_b200/ops/_build

.PHONY: all build rebuild test test-gpu sanitize sass bench wheel clean
