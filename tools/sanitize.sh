#!/bin/bash
# Race / memory checking (SURVEY 5.2: the reference has none).
#   tools/sanitize.sh gpu   -> compute-sanitizer memcheck + racecheck + synccheck over the single-GPU
#                              kernel tests (run it through gpurun; needs a GPU)
#   tools/sanitize.sh host  -> ThreadSanitizer build of the C++ host runtime + native unit / 4-process suites
#   tools/sanitize.sh apps <corpus.txt> <logreg.config>
#                           -> AddressSanitizer+UBSan+LeakSanitizer and ThreadSanitizer builds of the native
#                              applications, 2 ranks each (TSAN with one trainer thread: the trainers are
#                              Hogwild by design)
set -e
ROOT=$(cd "$(dirname "$0")/.." && pwd)
cd $ROOT
case "${1:-host}" in
gpu)
  mkdir -p gpurun_out
  for tool in memcheck racecheck synccheck; do
    timeout 1200 compute-sanitizer --tool $tool --error-exitcode 1 --log-file gpurun_out/sanitizer_$tool.log \
      python -m pytest tests/test_gpu_tables.py tests/test_gpu_get_gemm.py tests/test_gpu_kv_tables.py tests/test_gpu_hash_evict.py \
      tests/test_gpu_adam.py tests/test_gpu_ftrl.py tests/test_gpu_hierarchical_softmax.py tests/test_gpu_factorization_machine.py \
      tests/test_gpu_field_aware_factorization_machine.py tests/test_gpu_search_exact.py tests/test_gpu_graph_embedding.py -q -m gpu -x \
      -k "not 1048576 and (not search_exact or tiny or zero_query or empty_batch) and not sbm and not case7 and not case8" \
      > gpurun_out/sanitizer_$tool.out 2>&1; echo "compute-sanitizer $tool rc=$?"
    grep -E "ERROR SUMMARY|RACECHECK SUMMARY" gpurun_out/sanitizer_$tool.log | tail -2
  done
  ;;
host)
  OUT=build/tsan
  mkdir -p $OUT
  SRCS=$(find csrc/host -name '*.cpp' -not -path '*/tools/*' -not -path '*/apps/*')
  g++ -std=c++17 -O1 -g -fsanitize=thread -fPIC -pthread -fopenmp -Iinclude -Icsrc/host $SRCS csrc/host/tools/mv_test/main.cpp -o $OUT/mv_test_tsan -ldl
  TSAN_OPTIONS="halt_on_error=0 second_deadlock_stack=1" $OUT/mv_test_tsan unit 2>&1 | tee $OUT/unit.log | grep -E "PASS|FAIL|WARNING: ThreadSanitizer" | sort | uniq -c
  for s in array matrix kv; do
    TSAN_OPTIONS="halt_on_error=0" python tools/mvrun.py -n 3 -- $OUT/mv_test_tsan $s 2>&1 | tee $OUT/$s.log | grep -E "PASS|FAIL|WARNING: ThreadSanitizer" | sort | uniq -c
  done
  ;;
apps)
  CORPUS=${2:?corpus}; CONFIG=${3:?logreg config}
  SRCS=$(find csrc/host -name '*.cpp' -not -path '*/tools/*' -not -path '*/apps/*')
  for san in address,undefined thread; do
    tag=${san%%,*}; OUT=build/$tag; mkdir -p $OUT
    for app in wordembedding logreg; do
      g++ -std=c++17 -O1 -g -fsanitize=$san -fno-omit-frame-pointer -pthread -fopenmp -Iinclude -Icsrc/host \
        -Icsrc/host/apps/$app $SRCS csrc/host/apps/$app/*.cpp -o $OUT/${app}_$tag -ldl &
    done; wait
    export ASAN_OPTIONS=detect_leaks=1:halt_on_error=0 TSAN_OPTIONS=halt_on_error=0
    python tools/mvrun.py -n 2 -- $OUT/wordembedding_$tag -train_file $CORPUS -size 16 -epoch 2 -threads 1 \
      -min_count 1 -data_block_size 60000 -omp_threads=1 2>&1 | tee $OUT/wordembedding.log | grep -cE "Sanitizer|runtime error" || true
    python tools/mvrun.py -n 2 -- $OUT/logreg_$tag $CONFIG -omp_threads=1 2>&1 | tee $OUT/logreg.log | grep -cE "Sanitizer|runtime error" || true
  done
  ;;
esac
