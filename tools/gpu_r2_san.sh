#!/bin/bash
mkdir -p gpurun_out
timeout 900 python -m pytest tests/test_gpu_type_a.py tests/test_gpu_type_fd.py tests/test_gpu_shim.py -m gpu -q -x 2>&1 | tail -2
bash tools/gpu_sanitize.sh
timeout 300 python bench.py --steps 5 --warmup 3 --workload prod16 --configs none 2>/dev/null | python -c "
import json,sys; d=json.loads([l for l in sys.stdin if l.startswith('{')][-1]); print('prod16', round(d['value']), d['parity'], d['stage_ms'])"
