# Developer entry points (counterpart of the reference Makefile: `make test` / format).
PY ?= python

build:
	$(PY) -c "import __graft_entry__ as g; g.build()"

test: build
	$(PY) -m pytest tests/ -x -q -m "not gpu"

test-gpu: build
	$(PY) -m pytest tests/ -x -q -m "gpu and not multigpu"

test-multigpu: build
	$(PY) -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 -m pytest tests/test_multigpu.py -m multigpu -q

smoke: build
	$(PY) -c "import __graft_entry__ as g; g.smoke()"

bench: build
	$(PY) bench.py

sass:
	cuobjdump -sass torchacc_b200/_C.so | grep -oE "[HQ]GMMA[A-Z0-9.]*|UTMA[A-Z0-9.]*|UBLKCP[A-Z0-9.]*|USETMAXREG[A-Z0-9_.]*" | sort | uniq -c

# compute-sanitizer over the hand-written kernels (the reference has no sanitizer hooks at all, SURVEY 5.2):
# memcheck + synccheck on the stand-alone GEMM harness (every descriptor / TMA path, static and dynamic tile
# scheduling) and memcheck on the op-level numerics tests.
sanitize: build
	compute-sanitizer --tool memcheck --error-exitcode 1 build/gemm_test 3 0 1
	compute-sanitizer --tool synccheck --error-exitcode 1 build/gemm_test 2 0 1
	compute-sanitizer --tool memcheck --error-exitcode 1 $(PY) -m pytest tests/test_ops_gpu.py -q -m gpu -k "rmsnorm or swiglu or rope or cross_entropy or adamw"

# peer-memory collectives under the sanitizer on 2 GPUs: NCCL-free self check (NCCL's own kernels abort a synccheck run)
sanitize-multigpu: build
	$(PY) -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --no-python \
		compute-sanitizer --tool synccheck $(PY) tools/symm_selfcheck.py

.PHONY: build test test-gpu test-multigpu smoke bench sass sanitize sanitize-multigpu
