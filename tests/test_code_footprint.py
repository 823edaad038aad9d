"""Instruction footprint of one iteration of the sparse kernel.  Every block walks the range from
pass I1 to the accept pass once per iteration, four blocks per SM at different points of it; code
that does not fit the instruction caches is fetched again on every iteration.  tools/sass_footprint.py
prints the range by phase; this keeps it under a budget.  Needs nvcc (sm_90a cross-compile), no GPU."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tools'))
import sass_footprint                    # noqa: E402

BUDGET = 132 * 1024                      # bytes of the per-iteration range (parent: 192 KiB)


@pytest.fixture(scope='module')
def report():
    if not (os.path.exists(sass_footprint.NVCC) and os.path.exists(sass_footprint.NVDISASM)):
        pytest.skip('nvcc / nvdisasm not available')
    return sass_footprint.footprint()


def test_iteration_range_within_budget(report):
    assert report['range_bytes'] <= BUDGET, report['phases']


def test_kernel_keeps_occupancy(report):
    # 128 registers x 128 threads: four blocks per SM on config 2
    assert report['ptxas'].get('regs', 0) <= 128, report['ptxas']


def test_division_log_pow_out_of_line(report):
    names = ' '.join(report['callees'])
    for f in ('sp_div', 'sp_log', 'sp_pow'):
        assert f in names, names
