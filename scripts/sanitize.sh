# compute-sanitizer memcheck + synccheck on small shapes of every kernel family (on the GPU; ~2 min)
set -x
for cfg in "31 1024 1" "31 1024 1 enc_front=0" "31 1024 1 splitk=3" "16 768 1" "21 1024 1 splitk=2" "11 512 1" "15 1024 1" "12 1024 1" "13 768 1" "14 512 1"; do
  timeout 250 compute-sanitizer --tool memcheck --print-limit 3 --error-exitcode 7 python scripts/run_one.py $cfg 2>&1 | grep -E "ERROR SUMMARY|Invalid|Error|done|trap" | head -5
done
for cfg in "21 1024 1 epi_assist=0" "21 1024 1" "31 1024 1 splitk=3" "31 1024 1"; do
  timeout 250 compute-sanitizer --tool synccheck --print-limit 3 python scripts/run_one.py $cfg 2>&1 | grep -E "ERROR SUMMARY|Barrier error|done|trap|at ftsgemm" | head -4
done
