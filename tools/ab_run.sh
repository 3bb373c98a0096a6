#!/bin/bash
# One-call A/B on a GPU box.  Candidates are library build variants (csrc/Makefile `variants`: librcmarl_<name>.so,
# selected with RCMARL_LIB) and / or environment switches of the default library.
#   AB_LIBS="v0 p0"                        variants to compare with the default library
#   AB_ENVS="RCMARL_BALANCED_GRID=1"     switches to compare with the default settings
#   AB_TEST_LIBS="v0"                    variants to run the kernel + trainer GPU tests with
# For every candidate: gradient sums of fixed seeded inputs compared with the default's bit for bit (tools/ab_grad.py),
# CUDA-event timings of rcmarl_grad at the C2 shapes, and a short C2 bench.  Then the full GPU suite with the defaults.
cd "$(dirname "$0")/.."
P=$PWD/resilient-consensus-based-marl_b200/rcmarl
mkdir -p gpurun_out
bench_line() {
  timeout 150 python bench.py --steps 2 --warmup 1 --no-cpu-baseline --no-e2e --no-consensus 2>&1 | tail -1 \
    | python -c "import sys, json; d = json.loads(sys.stdin.read()); print('BENCH', d['ms_per_step'], d['value'], d['gpu_launches'], d['roofline']['regimes']['full_batch']['ms_per_launch'])"
}
echo "== default"
timeout 120 python tools/ab_grad.py dump gpurun_out/ab_base.npz 2>&1 | tail -3
bench_line
for v in $AB_LIBS; do
  echo "== library variant $v"
  RCMARL_LIB=$P/librcmarl_$v.so timeout 120 python tools/ab_grad.py dump gpurun_out/ab_$v.npz 2>&1 | tail -3
  python tools/ab_grad.py cmp gpurun_out/ab_base.npz gpurun_out/ab_$v.npz | tail -4
  RCMARL_LIB=$P/librcmarl_$v.so bench_line
done
i=0
for e in $AB_ENVS; do
  i=$((i + 1))
  echo "== switch $e"
  env "$e" timeout 120 python tools/ab_grad.py dump gpurun_out/ab_env$i.npz 2>&1 | tail -3
  python tools/ab_grad.py cmp gpurun_out/ab_base.npz gpurun_out/ab_env$i.npz | tail -4
  env "$e" bash -c "$(declare -f bench_line); bench_line"
done
for v in $AB_TEST_LIBS; do
  echo "== pytest kernels + trainer (library variant $v)"
  RCMARL_LIB=$P/librcmarl_$v.so timeout 300 python -m pytest tests/test_kernels_gpu.py tests/test_trainer_gpu.py -m gpu -q -x 2>&1 | tail -3
done
echo "== pytest (defaults)"
timeout 300 python -m pytest tests -m gpu -q -x 2>&1 | tail -3
timeout 120 python -c "import __graft_entry__ as g; g.smoke()" 2>&1 | tail -1
