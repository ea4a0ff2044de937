#!/bin/bash
# compute-sanitizer over the parity subset and the single-rank group path (memcheck, then racecheck on the
# private-histogram / fold / merge kernels).  Writes gpurun_out/sanitizer_{memcheck,racecheck}.txt
mkdir -p gpurun_out
SEL='ragged_sizes or nbins or special_values or constant_column or histogram_only or hist_u8 or unaligned or empty_inputs or memory_arrangement'
timeout 900 compute-sanitizer --tool memcheck --error-exitcode 1 python -m pytest tests/test_gpu_parity.py -q -k "$SEL" \
    tests/test_gpu_group.py::test_rank_group_one_rank_per_step_launch_count > gpurun_out/sanitizer_memcheck.txt 2>&1
echo "memcheck rc=$?"; tail -3 gpurun_out/sanitizer_memcheck.txt
# memcheck of the text dictionary codes (slot pass, shard merge, remap); its log goes to a temporary directory
codes_log="$(mktemp -d)/sanitizer_memcheck_text_codes.txt"
timeout 900 compute-sanitizer --tool memcheck --error-exitcode 1 python -m pytest tests/test_gpu_text_codes.py -q \
    > "$codes_log" 2>&1
echo "memcheck (text codes) rc=$? log=$codes_log"; tail -3 "$codes_log"
# memcheck of the feature matrix (validity pass, scan, write pass; every shape and refusal); its log goes to a temporary directory
features_log="$(mktemp -d)/sanitizer_memcheck_features.txt"
timeout 900 compute-sanitizer --tool memcheck --error-exitcode 1 python -m pytest tests/test_gpu_features.py -q \
    > "$features_log" 2>&1
echo "memcheck (features) rc=$? log=$features_log"; tail -3 "$features_log"
# memcheck of the NaiveBayes kernels (fit, transform, evaluate; every shape, cap and refusal); its log goes to a temporary directory
nb_log="$(mktemp -d)/sanitizer_memcheck_naive_bayes.txt"
timeout 1800 compute-sanitizer --tool memcheck --error-exitcode 1 python -m pytest tests/test_gpu_naive_bayes.py -q \
    > "$nb_log" 2>&1
echo "memcheck (naive bayes) rc=$? log=$nb_log"; tail -3 "$nb_log"
# memcheck of the refused cells over one GPU and every cut (the key's report and read-back); its log goes to a temporary directory
refused_log="$(mktemp -d)/sanitizer_memcheck_refused_cells.txt"
timeout 900 compute-sanitizer --tool memcheck --error-exitcode 1 python -m pytest tests/test_gpu_refused_cells.py -q \
    > "$refused_log" 2>&1
echo "memcheck (refused cells) rc=$? log=$refused_log"; tail -3 "$refused_log"
# memcheck of the LogisticRegression kernels (stats, loss / gradient, the binomial predict; every shape, cap and
# refusal); its log goes to a temporary directory
lr_log="$(mktemp -d)/sanitizer_memcheck_logistic.txt"
timeout 1800 compute-sanitizer --tool memcheck --error-exitcode 1 python -m pytest tests/test_gpu_logistic.py \
    tests/test_gpu_logistic_exact.py -q > "$lr_log" 2>&1
echo "memcheck (logistic) rc=$? log=$lr_log"; tail -3 "$lr_log"
# racecheck of k_lr_stats / k_lr_loss_grad (four shared-memory phases per tile) over every launch shape; its log goes to
# a temporary directory
lr_race_log="$(mktemp -d)/sanitizer_racecheck_logistic.txt"
timeout 1800 compute-sanitizer --tool racecheck --error-exitcode 1 python -m pytest tests/test_gpu_logistic_exact.py -q \
    -k "shape" > "$lr_race_log" 2>&1
echo "racecheck (logistic) rc=$? log=$lr_race_log"; tail -3 "$lr_race_log"
# memcheck and racecheck of the DecisionTree kernels (sort, distinct, rank, bin, every level route, predict, evaluate;
# the caps and refusals); their logs go to a temporary directory
dt_log="$(mktemp -d)/sanitizer_memcheck_tree.txt"
timeout 1800 compute-sanitizer --tool memcheck --error-exitcode 1 python -m pytest tests/test_gpu_tree.py -q > "$dt_log" 2>&1
echo "memcheck (tree) rc=$? log=$dt_log"; tail -3 "$dt_log"
dt_race_log="$(mktemp -d)/sanitizer_racecheck_tree.txt"
timeout 1800 compute-sanitizer --tool racecheck --error-exitcode 1 python -m pytest tests/test_gpu_tree.py -q \
    -k "route or edges" > "$dt_race_log" 2>&1
echo "racecheck (tree) rc=$? log=$dt_race_log"; tail -3 "$dt_race_log"
# memcheck and racecheck of the GBT kernels (every level route with 128-bit sums, update, predict, evaluate; the edges and
# refusals); their logs go to a temporary directory
gb_log="$(mktemp -d)/sanitizer_memcheck_gbt.txt"
timeout 1800 compute-sanitizer --tool memcheck --error-exitcode 1 python -m pytest tests/test_gpu_gbt.py -q > "$gb_log" 2>&1
echo "memcheck (gbt) rc=$? log=$gb_log"; tail -3 "$gb_log"
gb_race_log="$(mktemp -d)/sanitizer_racecheck_gbt.txt"
timeout 1800 compute-sanitizer --tool racecheck --error-exitcode 1 python -m pytest tests/test_gpu_gbt.py -q \
    -k "route or edges" > "$gb_race_log" 2>&1
echo "racecheck (gbt) rc=$? log=$gb_race_log"; tail -3 "$gb_race_log"
# memcheck and racecheck of the RandomForest kernels (every level route and tree batch, transform and evaluate with
# votes in registers and in the row's slice; the edges and refusals); their logs go to a temporary directory
rf_log="$(mktemp -d)/sanitizer_memcheck_rf.txt"
timeout 1800 compute-sanitizer --tool memcheck --error-exitcode 1 python -m pytest tests/test_gpu_rf.py -q > "$rf_log" 2>&1
echo "memcheck (rf) rc=$? log=$rf_log"; tail -3 "$rf_log"
rf_race_log="$(mktemp -d)/sanitizer_racecheck_rf.txt"
timeout 1800 compute-sanitizer --tool racecheck --error-exitcode 1 python -m pytest tests/test_gpu_rf.py -q \
    -k "route or edges" > "$rf_race_log" 2>&1
echo "racecheck (rf) rc=$? log=$rf_race_log"; tail -3 "$rf_race_log"
# memcheck of the number parser and the resident formatter on every entry point, without the million-row cases: a read
# past the last staged cell shows here (the CPU harness puts a NUL after it)
parse_log="$(mktemp -d)/sanitizer_memcheck_parse.txt"
timeout 900 compute-sanitizer --tool memcheck --error-exitcode 1 python -m pytest tests/test_gpu_parse.py -q -k "not million" \
    > "$parse_log" 2>&1
echo "memcheck (parse) rc=$? log=$parse_log"; tail -3 "$parse_log"
timeout 900 compute-sanitizer --tool racecheck --error-exitcode 1 python -m pytest tests/test_gpu_parity.py -q -k "ragged_sizes or nbins or hist_u8 or constant_column" \
    > gpurun_out/sanitizer_racecheck.txt 2>&1
echo "racecheck rc=$?"; tail -3 gpurun_out/sanitizer_racecheck.txt
