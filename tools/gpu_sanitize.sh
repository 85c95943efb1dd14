# compute-sanitizer memcheck over the kernels that changed in round 2 (BA chain, loop closure) and the loop-closure model tests (the -1-count header included)
set +e
export PYTHONUNBUFFERED=1
timeout 200 compute-sanitizer --tool memcheck --print-limit 8 python -m pytest tests/test_gpu_ba.py -x -q -p no:cacheprovider -k "golden or duplicate" 2>&1 | grep -E "ERROR SUMMARY|Invalid|passed|failed|at .*\(|========= " | head -20
timeout 150 compute-sanitizer --tool memcheck --print-limit 8 python -m pytest tests/test_gpu_loopclosure.py -x -q -p no:cacheprovider -k "wire_format" 2>&1 | grep -E "ERROR SUMMARY|Invalid|passed|failed|at .*\(|========= " | head -20
timeout 600 compute-sanitizer --tool memcheck --print-limit 8 python -m pytest tests/test_gpu_loopclosure_model.py -x -q -p no:cacheprovider -k "not largest" 2>&1 | grep -E "ERROR SUMMARY|Invalid|passed|failed|at .*\(|========= " | head -20
