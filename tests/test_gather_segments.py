"""The sparse kernel's factorisation gather by column segments (omg_sp_host.cuh, omg_sp.cuh):
up to SP_GQ consecutive entries of a column share one record per source supernode.

From the host tables: every entry reads its own pair list back from its segment's records, in
list order (seg-mismatch=0 on the structure line), for config 2 and every synthetic family.
From the emulated kernel: the default build and a build with one entry per segment (SP_GQ=1,
the record-per-entry gather) give bit-identical x, lam_g, f, statuses and iteration counts."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import ipm_c

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import emu_support                       # noqa: E402
import synthetic_kkt as sk               # noqa: E402

Q1_NAME = 'libomgb200_emu_q1.so'
Q1_LIB = os.path.join(emu_support.EMU_DIR, '_build', Q1_NAME)
FAMILIES = sk.families()


@pytest.fixture(scope='module')
def emu():
    if not ipm_c.available():
        pytest.skip('C oracle not built')
    saved = emu_support.activate()
    yield
    emu_support.restore(saved)


def _build_q1():
    emu_support.build()
    if not os.path.exists(Q1_LIB) or os.path.getmtime(Q1_LIB) < os.path.getmtime(emu_support.EMU_LIB):
        subprocess.check_call([os.path.join(emu_support.EMU_DIR, 'build.sh'), Q1_NAME, '-DSP_GQ=1'])


def _solve(lib, tb, X0, P):
    from omg_tools_b200.solver import b200
    saved = b200._lib
    b200._lib = lib
    try:
        slv = b200.B200Solver(tb, {})
        return slv.structure, slv.solve_batch(X0, P)
    finally:
        b200._lib = saved


def _config2_tables():
    from omg_tools_b200 import scenarios as sc
    pr = sc.config2(build_solver=False)
    X0, P = sc.instance_data(pr, 3, jitter=0.2, seed=11)
    return pr.father.tables, X0, P


def test_segments_reproduce_every_pair_list(emu):
    from omg_tools_b200.solver import b200
    tables = [('config2', _config2_tables()[0])] + [(n, FAMILIES[n]().tb) for n in FAMILIES]
    seen = 0
    for name, tb in tables:
        s = b200.B200Solver(tb, {}).structure
        if s.startswith('envelope'):
            continue
        cnt = sk.parse_counters(s)
        assert cnt['seg-mismatch'] == 0, (name, s)
        assert cnt['segments'] <= cnt['nnz(L)'], (name, s)
        seen += cnt['segments'] > 0
    assert seen > 20


@pytest.mark.parametrize('name', ['config2', 'arrow', 'fan-wide'])
def test_segments_match_one_entry_per_segment_bit_for_bit(emu, name):
    """Config 2 (58 % of its records gather into the dense root) and two families with long
    lists: the root gather of 'arrow' and the 40-source lists of 'fan-wide'."""
    from omg_tools_b200.solver import b200
    _build_q1()
    if name == 'config2':
        tb, X0, P = _config2_tables()
    else:
        c = FAMILIES[name]()
        tb, X0, P = c.tb, c.X0, c.P
    s_q, res_q = _solve(b200._lib, tb, X0, P)
    s_1, res_1 = _solve(b200.bind(C.CDLL(Q1_LIB)), tb, X0, P)
    cq, c1 = sk.parse_counters(s_q), sk.parse_counters(s_1)
    assert c1['segments'] > cq['segments'] and c1['seg-records'] > cq['seg-records'], (s_q, s_1)
    assert cq['max-seg-sources'] >= c1['max-seg-sources'] == cq['max-gather'], (s_q, s_1)
    assert cq['pairs'] == c1['pairs'], (s_q, s_1)          # pairs= counts the record-per-entry slots
    assert (res_q['status'] == 0).all()
    for key in ('x', 'lam_g', 'f', 'status', 'iters'):
        assert np.array_equal(res_q[key], res_1[key]), key
