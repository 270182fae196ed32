#!/bin/bash
# Round-end style check on an H100: GPU parity suite, smoke(), both bench arms.
cd "${GRAFT_REPO_ROOT:-$(dirname "$0")/..}" || exit 1
mkdir -p gpurun_out
(timeout 900 python -m pytest tests -q -m gpu 2>&1 | tail -3) > gpurun_out/check_pytest.txt
python -c "import __graft_entry__ as g; g.smoke()" > gpurun_out/check_smoke.txt 2>&1
(timeout 600 python bench.py --impl reference --steps 3 --warmup 1 2> gpurun_out/check_bench_ref.err | tail -1) > gpurun_out/check_bench_ref.json
(timeout 900 python bench.py --steps 10 --warmup 3 2> gpurun_out/check_bench.err | tail -1) > gpurun_out/check_bench.json
tail -1 gpurun_out/check_pytest.txt; cat gpurun_out/check_smoke.txt; cut -c1-260 gpurun_out/check_bench.json; cut -c1-200 gpurun_out/check_bench_ref.json
