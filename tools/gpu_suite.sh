#!/bin/bash
# One gpurun call = everything we want from a box. Usage: tools/gpu_suite.sh [NGPU] [stage...]
# Output goes to gpurun_out/ (merged back into the repo by gpurun).
NG=${1:-1}; shift
STAGES=${@:-"info test smoke bench mp ncu"}
mkdir -p gpurun_out
export MVB200_NO_BUILD=1
PORT=29511
for s in $STAGES; do
case $s in
info)
  nvidia-smi --query-gpu=index,name,clocks.sm,clocks.max.sm,power.draw,memory.total --format=csv > gpurun_out/info.txt 2>&1
  nvidia-smi topo -m >> gpurun_out/info.txt 2>&1
  ;;
test)
  timeout 900 python -m pytest tests -m gpu -x -q > gpurun_out/pytest_gpu.log 2>&1; echo "pytest rc=$?" | tee -a gpurun_out/pytest_gpu.log
  tail -15 gpurun_out/pytest_gpu.log
  ;;
smoke)
  timeout 300 python -c "import __graft_entry__ as g; g.smoke()" > gpurun_out/smoke.log 2>&1; echo "smoke rc=$?"; tail -3 gpurun_out/smoke.log
  ;;
bench)
  timeout 600 python bench.py --steps 10 --warmup 3 > gpurun_out/bench_n1.json 2> gpurun_out/bench_n1.err; echo "bench rc=$?"; cat gpurun_out/bench_n1.json; tail -5 gpurun_out/bench_n1.err
  ;;
mp)
  if [ "$NG" -gt 1 ]; then
    timeout 400 python -m torch.distributed.run --nnodes=1 --nproc-per-node $NG --master-addr 127.0.0.1 --master-port $PORT tests/mp_device_check.py > gpurun_out/mp_check.log 2>&1; echo "mp rc=$?"; grep -E "PASS|FAIL|Error|error" gpurun_out/mp_check.log | head -20
    timeout 400 python -m torch.distributed.run --nnodes=1 --nproc-per-node $NG --master-addr 127.0.0.1 --master-port $((PORT+1)) bench.py --gpus $NG --steps 10 --warmup 3 > gpurun_out/bench_n$NG.json 2> gpurun_out/bench_n$NG.err; echo "bench$NG rc=$?"; cat gpurun_out/bench_n$NG.json; tail -5 gpurun_out/bench_n$NG.err
  fi
  ;;
ncu)
  timeout 600 ncu --metrics gpu__time_duration.sum --clock-control none -c 60 --csv --log-file gpurun_out/launches.csv python bench.py --steps 2 --warmup 3 > gpurun_out/ncu_launches.log 2>&1; echo "launches rc=$?"
  ;;
ncu_dense)
  timeout 600 ncu --set full --clock-control none --import-source on -k regex:"add_dense_fused|get_dense" -c 4 -f -o gpurun_out/dense python -c "
import torch, multiverso_b200 as mv
mv.init(); t = mv.MatrixTable(1000000, 512, 'float32', updater='sgd'); d = torch.ones(512000000, device='cuda')
t.add(d); t.get(); t.add(d); t.get(); mv.shutdown()" > gpurun_out/ncu_dense.log 2>&1; echo "ncu_dense rc=$?"
  ;;
extra)
  if [ "$NG" -gt 1 ]; then L="python -m torch.distributed.run --nnodes=1 --nproc-per-node $NG --master-addr 127.0.0.1 --master-port $((PORT+5))"; else L="python"; fi
  timeout 300 $L bench/matrix_bw.py > gpurun_out/matrix_bw.log 2>&1; echo "matrix_bw rc=$?"; grep '^{' gpurun_out/matrix_bw.log | tail -1 | cut -c1-600
  timeout 300 $L bench/matrix_bw.py --array-gb 4 --updater momentum_sgd > gpurun_out/array_bw.log 2>&1; echo "array_bw rc=$?"; grep '^{' gpurun_out/array_bw.log | tail -1 | cut -c1-600
  timeout 300 $L bench/logreg_sparse.py > gpurun_out/logreg_sparse.log 2>&1; echo "logreg_sparse rc=$?"; grep '^{' gpurun_out/logreg_sparse.log | tail -1 | cut -c1-400
  ;;
sanitize)
  timeout 900 compute-sanitizer --tool memcheck --error-exitcode 1 --log-file gpurun_out/sanitizer_memcheck.log python -m pytest tests/test_gpu_tables.py tests/test_gpu_get_gemm.py -q -m gpu -x -k "not 1048576 and not 1000-1000-512 and not 2048-300-300" > gpurun_out/sanitizer_memcheck.out 2>&1; echo "memcheck rc=$?"; grep -E "ERROR SUMMARY" gpurun_out/sanitizer_memcheck.log | tail -3; tail -2 gpurun_out/sanitizer_memcheck.out
  ;;
replica)
  L="python -m torch.distributed.run --nnodes=1 --nproc-per-node $NG --master-addr 127.0.0.1 --master-port $((PORT+7))"
  timeout 300 $L bench/matrix_bw.py --replica > gpurun_out/matrix_bw_replica.log 2>&1; echo "matrix_bw replica rc=$?"; grep '^{' gpurun_out/matrix_bw_replica.log | tail -1 | cut -c1-700
  ;;
gemm)
  if [ "$NG" -gt 1 ]; then L="python -m torch.distributed.run --nnodes=1 --nproc-per-node $NG --master-addr 127.0.0.1 --master-port $((PORT+6))"; else L="python"; fi
  timeout 300 $L bench/get_gemm.py > gpurun_out/get_gemm.log 2>&1; echo "get_gemm rc=$?"; grep '^\[' gpurun_out/get_gemm.log | tail -1 | cut -c1-900
  ;;
ncu_gemm)
  timeout 400 ncu --set full --clock-control none --import-source on -k regex:get_gemm_fused -s 2 -c 1 -f -o gpurun_out/get_gemm python bench/get_gemm.py --shapes 4096x65536x512 --iters 2 > gpurun_out/ncu_get_gemm.log 2>&1; echo "ncu_gemm rc=$?"
  ;;
allreduce)
  timeout 300 python -m torch.distributed.run --nnodes=1 --nproc-per-node $NG --master-addr 127.0.0.1 --master-port $((PORT+9)) bench/allreduce.py > gpurun_out/allreduce.log 2>&1; echo "allreduce rc=$?"; grep '^\[' gpurun_out/allreduce.log | tail -1 | python -c "
import sys,json
for l in sys.stdin:
    for r in json.loads(l): print({k:(round(v,1) if isinstance(v,float) else v) for k,v in r.items()})"
  ;;
perf)
  if [ "$NG" -gt 1 ]; then L="python -m torch.distributed.run --nnodes=1 --nproc-per-node $NG --master-addr 127.0.0.1 --master-port $((PORT+8))"; else L="python"; fi
  timeout 300 $L bench/matrix_perf.py > gpurun_out/matrix_perf.log 2>&1; echo "matrix_perf dense rc=$?"; grep '^{' gpurun_out/matrix_perf.log | tail -1 | cut -c1-500
  timeout 300 $L bench/matrix_perf.py --sparse > gpurun_out/matrix_perf_sparse.log 2>&1; echo "matrix_perf sparse rc=$?"; grep '^{' gpurun_out/matrix_perf_sparse.log | tail -1 | cut -c1-500
  ;;
win)
  # round 2: window-batched K7: numerics, 1-GPU bench, ncu
  timeout 600 python -m pytest tests/test_gpu_wordembedding.py -x -q > gpurun_out/pytest_we.log 2>&1; echo "pytest we rc=$?"; tail -8 gpurun_out/pytest_we.log
  timeout 300 python bench.py --steps 10 --warmup 3 > gpurun_out/bench_n1_win.json 2> gpurun_out/bench_n1_win.err; echo "bench win rc=$?"; cut -c1-700 gpurun_out/bench_n1_win.json; tail -3 gpurun_out/bench_n1_win.err
  timeout 600 ncu --set full --clock-control none --import-source on -k regex:sgns_win -s 3 -c 1 -f -o gpurun_out/sgns_win python bench.py --steps 2 --warmup 3 --no-table-bw > gpurun_out/ncu_sgns_win.log 2>&1; echo "ncu rc=$?"; tail -3 gpurun_out/ncu_sgns_win.log
  ;;
cap)
  # hot-row step cap sweep: loss after the same number of blocks
  timeout 600 python -m pytest tests/test_gpu_wordembedding.py -x -q > gpurun_out/pytest_we.log 2>&1; echo "pytest we rc=$?"; tail -5 gpurun_out/pytest_we.log
  for st in ${CAP_STEPS:-6 22}; do
  for c in ${CAPS:-32 64 128 256 512}; do
    MVB_WE_HOT_CAP=$c timeout 300 python bench.py --steps $st --warmup 3 --no-table-bw > gpurun_out/cap_${c}_s$st.json 2>/dev/null; python -c "import json;d=json.load(open('gpurun_out/cap_${c}_s$st.json'));print('cap $c steps $st', round(d['value']/1e6,1), d['config']['loss_per_pair'])"
  done
  done
  ;;
blk)
  # round 2: device-side block protocol: 1-GPU kernel tests, then (NG>1) multi-GPU scenarios + bench
  timeout 600 python -m pytest tests/test_gpu_we_block.py tests/test_gpu_wordembedding.py -x -q > gpurun_out/pytest_blk.log 2>&1; echo "pytest blk rc=$?"; tail -6 gpurun_out/pytest_blk.log
  if [ "$NG" -gt 1 ]; then
    timeout 500 python -m torch.distributed.run --nnodes=1 --nproc-per-node $NG --master-addr 127.0.0.1 --master-port $PORT tests/mp_device_check.py async > gpurun_out/mp_check_async.log 2>&1; echo "mp async rc=$?"; grep -E "PASS|FAIL|Error|error" gpurun_out/mp_check_async.log | head -12
    timeout 400 python -m torch.distributed.run --nnodes=1 --nproc-per-node $NG --master-addr 127.0.0.1 --master-port $((PORT+1)) bench.py --gpus $NG --steps 10 --warmup 3 > gpurun_out/bench_n$NG.json 2> gpurun_out/bench_n$NG.err; echo "bench$NG rc=$?"; cut -c1-1500 gpurun_out/bench_n$NG.json; tail -5 gpurun_out/bench_n$NG.err
  fi
  ;;
r2n8)
  # round 2, one multi-GPU call: scenarios (async + sync), headline bench, dense Get bulk experiment
  for w in async sync; do
    timeout 500 python -m torch.distributed.run --nnodes=1 --nproc-per-node $NG --master-addr 127.0.0.1 --master-port $((PORT+20)) tests/mp_device_check.py $w > gpurun_out/mp_check_${w}_n$NG.log 2>&1; echo "mp $w rc=$?"; grep -cE "PASS" gpurun_out/mp_check_${w}_n$NG.log; grep -E "FAIL|Error|Traceback" gpurun_out/mp_check_${w}_n$NG.log | head -5 | cut -c1-600
  done
  timeout 500 python -m torch.distributed.run --nnodes=1 --nproc-per-node $NG --master-addr 127.0.0.1 --master-port $((PORT+21)) bench.py --gpus $NG --steps 20 --warmup 5 > gpurun_out/bench_n$NG.json 2> gpurun_out/bench_n$NG.err; echo "bench$NG rc=$?"; grep '^{' gpurun_out/bench_n$NG.json | cut -c1-1200; tail -3 gpurun_out/bench_n$NG.err
  L="python -m torch.distributed.run --nnodes=1 --nproc-per-node $NG --master-addr 127.0.0.1 --master-port $((PORT+23))"
  for v in 0 1; do
    MVB_GET_BULK=$v timeout 300 $L bench/matrix_bw.py > gpurun_out/matrix_bw_bulk${v}_n$NG.log 2>&1; echo "matrix_bw MVB_GET_BULK=$v rc=$?"; grep '^{' gpurun_out/matrix_bw_bulk${v}_n$NG.log | tail -1 | cut -c1-700
  done
  ;;
r2final)
  # round 2 final multi-GPU call: config-5 stress, headline bench
  L="python -m torch.distributed.run --nnodes=1 --nproc-per-node $NG --master-addr 127.0.0.1 --master-port $((PORT+31))"
  timeout 400 $L bench/array_async_stress.py > gpurun_out/array_async_stress_n$NG.log 2>&1; echo "stress rc=$?"; grep '^{' gpurun_out/array_async_stress_n$NG.log | tail -1 | cut -c1-900
  timeout 500 python -m torch.distributed.run --nnodes=1 --nproc-per-node $NG --master-addr 127.0.0.1 --master-port $((PORT+32)) bench.py --gpus $NG --steps 20 --warmup 5 > gpurun_out/bench_n$NG.json 2> gpurun_out/bench_n$NG.err; echo "bench$NG rc=$?"; grep '^{' gpurun_out/bench_n$NG.json | cut -c1-400; tail -3 gpurun_out/bench_n$NG.err
  ;;
refarm)
  timeout 1500 python bench.py --impl reference --gpus 1 > gpurun_out/bench_ref_n1.json 2> gpurun_out/bench_ref_n1.err; echo "ref rc=$?"; cut -c1-300 gpurun_out/bench_ref_n1.json
  ;;
bulk)
  # EXPERIMENT: dense Get through the bulk-copy engine (MVB_GET_BULK=1) -- correctness first, then time it
  MVB_GET_BULK=1 timeout 600 python -m pytest tests/test_gpu_tables.py -q -m gpu -x -k "array or matrix" > gpurun_out/bulk_pytest.log 2>&1; echo "bulk pytest rc=$?"; tail -2 gpurun_out/bulk_pytest.log
  if [ "$NG" -gt 1 ]; then L="python -m torch.distributed.run --nnodes=1 --nproc-per-node $NG --master-addr 127.0.0.1 --master-port $((PORT+11))"; else L="python"; fi
  for v in 0 1; do
    MVB_GET_BULK=$v timeout 300 $L bench/matrix_bw.py > gpurun_out/matrix_bw_bulk$v.log 2>&1; echo "matrix_bw MVB_GET_BULK=$v rc=$?"; grep '^{' gpurun_out/matrix_bw_bulk$v.log | tail -1 | cut -c1-500
  done
  ;;
nvls_cpp)
  # C++ device runtime, NVLS all-reduce on VMM / multicast-bound staging (csrc/device_rt/vmm.cpp, -device_nvls):
  # written after round 2's GPU budget was spent, NOT yet executed -- run this first (needs >= 2 GPUs; from 4 the
  # `auto` setting 1 also takes the NVLS path).  A platform without multicast objects must pass on the fallback.
  if [ "$NG" -gt 1 ]; then
    for mode in 2 1; do
      timeout 260 python tools/mvrun.py -n $NG --timeout 200 -- build/bin/mv_device_test aggregate -device_nvls=$mode > gpurun_out/devrt_nvls${mode}_n$NG.log 2>&1; echo "mv_device_test aggregate -device_nvls=$mode rc=$?"; grep -E "PASS|FAIL|EXPECT|NVLS" gpurun_out/devrt_nvls${mode}_n$NG.log | head -12
    done
  else echo "nvls_cpp needs > 1 GPU"; fi
  ;;
devrt)
  # native C++ device runtime scenarios (BSP + async) and the native GPU wordembedding application
  if [ "$NG" -gt 1 ]; then L="python tools/mvrun.py -n $NG --timeout 200 --"; else L=""; fi
  for sync in true false; do
    timeout 260 $L build/bin/mv_device_test all -sync=$sync > gpurun_out/devrt_n${NG}_sync_$sync.log 2>&1; echo "mv_device_test sync=$sync rc=$?"; grep -E "PASS|FAIL|EXPECT" gpurun_out/devrt_n${NG}_sync_$sync.log | head -12
  done
  timeout 200 $L python tools/check_gpu_c_api.py > gpurun_out/gpu_c_api_n$NG.log 2>&1; echo "gpu c api rc=$?"; grep -E "gpu c api ok|Error|FATAL" gpurun_out/gpu_c_api_n$NG.log | head -8
  timeout 200 $L build/bin/mv_device_test bench -sync=true > gpurun_out/devrt_bench_n$NG.log 2>&1; echo "mv_device_test bench rc=$?"; grep '^{' gpurun_out/devrt_bench_n$NG.log | head -8
  python - <<'PY'
import numpy as np
rng = np.random.default_rng(0)
with open("gpurun_out/topics.txt", "w") as f:
    for _ in range(20000):
        t = rng.integers(20); ws = rng.integers(50, size=rng.integers(5, 20))
        f.write(" ".join(f"t{t}w{w}" for w in ws) + "\n")
PY
  python - <<'PY'
import numpy as np
rng = np.random.default_rng(1)
D, C, N = 20, 4, 6000
Wt = rng.normal(size=(C, D)); X = rng.normal(size=(N, D)); y = (X @ Wt.T).argmax(1)
for name, lo, hi in (("train", 0, 5000), ("test", 5000, 6000)):
    with open(f"gpurun_out/lr_{name}.txt", "w") as f:
        for xi, yi in zip(X[lo:hi], y[lo:hi]):
            f.write(str(int(yi)) + " " + " ".join("%.4f" % v for v in xi) + "\n")
for ps in ("false", "true"):
    open(f"gpurun_out/lr_ps_{ps}.config", "w").write(f"""input_size=20
output_size=4
objective_type=softmax
regular_type=L2
updater_type=sgd
learning_rate=0.5
train_epoch=3
minibatch_size=20
use_ps={ps}
pipeline=true
sync_frequency=2
train_file=gpurun_out/lr_train.txt
test_file=gpurun_out/lr_test.txt
output_file=gpurun_out/lr_{ps}.out
output_model_file=gpurun_out/lr_{ps}.model
""")
PY
  timeout 200 build/bin/logreg_gpu gpurun_out/lr_ps_false.config > gpurun_out/lr_gpu_local.log 2>&1; echo "logreg_gpu local rc=$?"; grep '^{' gpurun_out/lr_gpu_local.log | cut -c1-300
  timeout 200 $L build/bin/logreg_gpu gpurun_out/lr_ps_true.config > gpurun_out/lr_gpu_ps_n$NG.log 2>&1; echo "logreg_gpu ps rc=$?"; grep '^{' gpurun_out/lr_gpu_ps_n$NG.log | head -8 | cut -c1-300
  timeout 300 $L build/bin/wordembedding_gpu -train_file gpurun_out/topics.txt -output gpurun_out/topics_vec.txt -size 32 -cbow 0 -negative 5 -epoch 3 -min_count 1 -data_block_size 300000 > gpurun_out/we_gpu_n$NG.log 2>&1; echo "wordembedding_gpu rc=$?"; grep '^{' gpurun_out/we_gpu_n$NG.log | head -8 | cut -c1-400
  ;;
probe)
  timeout 300 python -m torch.distributed.run --nnodes=1 --nproc-per-node $NG --master-addr 127.0.0.1 --master-port $((PORT+2)) tools/probe_symm.py > gpurun_out/probe.log 2>&1; echo "probe rc=$?"; tail -20 gpurun_out/probe.log
  ;;
esac
done
ls -la gpurun_out | head -40
