#!/bin/bash
# Quick GPU check after a kernel change: parity + node + stress tests, drop-in timing, headline bench.
cd /root/repo
( timeout 1800 python -m pytest tests/test_gpu_node.py tests/test_gpu_parity.py tests/test_gpu_stress.py -m gpu -x -q 2>&1 | tail -6 )
bash scripts/dropin_time.sh sboxgates_gpu 2>&1 | grep -v "^\[sbg\] start-up" | cut -c1-330
