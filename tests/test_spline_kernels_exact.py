"""The four spline kernels against exact rational arithmetic (tests/spline_exact.py), at the shapes,
knots and abscissae where they could go wrong, and the argument checks of their C calls.

Each family runs the kernel source on the CPU (tools/cpu_emu) without a mark and on the device
with the gpu mark.  Every entry is compared with its exact value within a bound derived from the
exact terms (spline_exact: k u sum |w| |q|, u = 2^-53), never a fixed tolerance, so a kernel that is
off by more than its own rounding fails.  Worst error / bound ratios measured (CPU emulation / H100
SXM; they differ by the device's FMA contraction):

* omg_eval_batch (test_eval_*): degrees 0..8 at L = p + 1, a middle L and 48; uniform, random,
  repeated (multiplicity 2..p) and jump (p + 1) interior knots, spans [0, 1], [-2.5, 7] and
  [1e3, 1e3 + 0.75]; the ends, every distinct knot and one ulp either side of it, random points
  and points outside the span (exactly 0); n_der 1 .. min(4, p + 1); scales 1e-3 .. 1e3; 1, 64 and
  65 columns; 1, 64, 65 and 203 points; blocks of different (L, p) in one call; 48 KB of derivative
  coefficients accepted, 8 bytes more rejected.  k = 4 (L + p).  Worst ratio 0.133 / 0.110.
* omg_shift_free_batch (test_shift_free_*): degrees 1..8, L at and around the thresholds 26, 33, 43
  of S = floor(128 / L) and at 48, uniform, random and repeated old knots, several blocks of
  different L per call, the T sweep of test_batch_mpc_freeT.py over both branches of the rule;
  result against the exact M c within k u max|c| sum_k |M_ik|, k = 4 (L + p).  A handle with
  n = 1250 makes the shared memory exceed 48 KB (the opt-in branch).  Bit-identical under the
  emulator's reverse and random schedules.  Worst ratio 0.649 / 0.693.
* omg_sample_batch / omg_shift_batch (test_fixed_rows_*): exact basis rows rounded to double and T
  matrices of spline_extra at L up to 48, n > 128, ns nc and L nc above 128, several blocks; against
  the exact dot product within 4 L u sum |a_i b_i|.  Worst ratio 0.054 / 0.038.  An x row above 48 KB
  (n = 7000) runs through the opt-in, one above 227 KB is rejected.
"""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import emu_support                       # noqa: E402
import spline_exact as se                # noqa: E402
import synthetic_kkt as sk               # noqa: E402
from omg_tools_b200.solver import b200   # noqa: E402

DT = 0.5
# test_batch_mpc_freeT.T_SWEEP: both branches of the rule (T < 2 dt: u = T - dt, target = T)
T_SWEEP = [DT + 1e-9, DT + 1e-4, 0.7, 2 * DT - 1e-9, 2 * DT + 1e-9, 2 * DT + 1e-4, 1.6, 3.7, 10., 24.]
T_OUTSIDE = [0.3, DT, 2 * DT]
WORST = {}


@pytest.fixture(scope='module')
def emu():
    saved = emu_support.activate()
    yield b200._lib
    emu_support.restore(saved)


@pytest.fixture(scope='module', autouse=True)
def _report():
    yield
    print('\nworst error / bound: ' + ', '.join('%s %.3g' % kv for kv in sorted(WORST.items())))


def _torch(a, device):
    import torch
    return torch.tensor(np.ascontiguousarray(a), device=device)


def _ratio(family, err, bound):
    """Largest err / bound, with err == 0 required where the bound is 0; recorded per family."""
    err, bound = np.asarray(err, dtype=float), np.asarray(bound, dtype=float)
    assert np.all(err[bound == 0] == 0), family
    r = float((err[bound > 0] / bound[bound > 0]).max()) if np.any(bound > 0) else 0.
    WORST[family] = max(WORST.get(family, 0.), r)
    return r


def _knots(kind, p, L, rng, span=(0., 1.)):
    """L + p + 1 clamped knots on span: interior knots uniform, random, with one knot of
    multiplicity m (kind ('mult', m)) or p + 1 (a jump of the function)."""
    a, b = span
    n_in = L - p - 1
    if kind == 'uniform' or n_in == 0:
        inner = np.linspace(a, b, n_in + 2)[1:-1]
    elif kind == 'random':
        inner = np.sort(rng.uniform(a, b, n_in))
    else:
        m = min(kind[1], n_in)
        rest = np.sort(rng.uniform(a, b, n_in - m))
        inner = np.sort(np.r_[rest, np.full(m, a + 0.4375 * (b - a))])
    return np.r_[np.full(p + 1, a), inner, np.full(p + 1, b)]


def _points(knots, n_pts, rng):
    """The ends, every distinct knot and one ulp either side, points outside the span, then
    random points inside, n_pts in all (the special ones first, cut to n_pts)."""
    a, b = knots[0], knots[-1]
    u = np.unique(knots)
    special = np.r_[a, b, u, np.nextafter(u, -np.inf), np.nextafter(u, np.inf), a - 1., b + 0.5, -1e300]
    pts = np.r_[special, rng.uniform(a, b, max(0, n_pts - len(special)))]
    return pts[:n_pts] if n_pts >= 3 else np.array([b, a, a - 1.])[:n_pts]


_ROWS = {}


def _basis_row(knots, p, d, x):
    """Exact basis row of the d-th derivative (degree p - d on knots[d:-d]) at x, cached."""
    key = (knots.tobytes(), p, d, float(x))
    if key not in _ROWS:
        _ROWS[key] = se.basis(list(knots)[d:len(knots) - d], p - d, x)
    return _ROWS[key]


def _exact_eval(blocks, X, tau, scale, n_der):
    """Exact out[b] of omg_eval_batch and the bounds, for the instances b of X."""
    vals, bnds = [], []
    for b in range(X.shape[0]):
        v_b, e_b = [], []
        s = se.fr(scale[b])
        for off, L, nc, p, knots in blocks:
            kb = 4 * (L + p)
            rows = {d: [_basis_row(knots, p, d, x) for x in tau[b]] for d in range(n_der)}
            for c in range(nc):
                col = X[b, off + c * L:off + (c + 1) * L]
                q = se.derivative_coeffs(knots, p, col, n_der)
                qa = se.derivative_coeffs(knots, p, col, n_der, magnitude=True)
                for j in range(len(tau[b])):
                    for d in range(n_der):
                        w = rows[d][j]
                        sd = s ** d
                        v_b.append(sum((wi * qi for wi, qi in zip(w, q[d]) if wi), se.F(0)) / sd)
                        e_b.append(float(kb * se.U * sum((wi * qi for wi, qi in zip(w, qa[d]) if wi), se.F(0)) / sd))
        vals.append(v_b)
        bnds.append(e_b)
    return vals, np.array(bnds)


def _check_eval(blocks, B, n_pts, n_der, device, rng, family, check=None):
    n = max(off + L * nc for off, L, nc, _, _ in blocks) + 3
    X = rng.standard_normal((B, n)) * 10. ** rng.uniform(-2, 2, (B, 1))
    pts = _points(np.concatenate([blk[4] for blk in blocks]), n_pts, rng)
    tau = np.array([rng.permutation(pts) for _ in range(B)])
    scale = 10. ** np.linspace(-3, 3, B) if B > 1 else np.array([1e-3])
    out = b200.eval_batch(_torch(X, device), blocks, _torch(tau, device), _torch(scale, device),
                          n_der).cpu().numpy()
    assert out.shape == (B, sum(blk[2] for blk in blocks) * n_pts * n_der)
    check = np.arange(B) if check is None else check
    vals, bnds = _exact_eval(blocks, X[check], tau[check], scale[check], n_der)
    err = np.array([[float(abs(se.F(g) - v)) for g, v in zip(out[b], vb)] for b, vb in zip(check, vals)])
    r = _ratio(family, err, bnds)
    assert r <= 1., (family, r)
    # outside the span every value is exactly 0
    for b in check:
        o = 0
        for off, L, nc, p, knots in blocks:
            outside = (tau[b] < knots[0]) | (tau[b] > knots[-1])
            blk = out[b, o:o + nc * n_pts * n_der].reshape(nc, n_pts, n_der)
            assert np.all(blk[:, outside, :] == 0.), family
            o += nc * n_pts * n_der
    return r


def _degree_blocks(p, rng):
    """Blocks of degree p: L = p + 1 (no interior knot), a middle L and 48, on each knot kind."""
    mid = (p + 1 + 48) // 2
    kinds = ['uniform', 'random'] + [('mult', m) for m in range(2, p + 1)] + [('mult', p + 1)]
    spans = [(0., 1.), (-2.5, 7.), (1e3, 1e3 + 0.75)]
    blocks, off = [], 0
    for i, (L, kind) in enumerate([(p + 1, 'uniform'), (mid, kinds[1 % len(kinds)]), (48, kinds[-1])] +
                                  [(mid, k) for k in kinds[2:-1]] + [(48, 'uniform')]):
        blocks.append((off, L, 1, p, _knots(kind, p, L, rng, spans[i % 3])))
        off += L
    return blocks


def _run_eval_degree(p, device, B):
    rng = np.random.default_rng(100 + p)
    blocks = _degree_blocks(p, rng)
    for n_der in range(1, min(4, p + 1) + 1):
        for blk in blocks:
            _check_eval([blk], B, 3 * len(np.unique(blk[4])) + 6, n_der, device, rng, 'eval')
    return WORST['eval']


@pytest.mark.parametrize('p', range(9))
def test_eval_degrees(emu, p):
    """Degrees 0..8, L = p + 1, middle and 48, every knot kind, every n_der up to min(4, p + 1),
    three instances with scales 1e-3, 1, 1e3 (and B = 1)."""
    print('p=%d worst ratio %.3g' % (p, _run_eval_degree(p, 'cpu', 3)))
    rng = np.random.default_rng(p)
    _check_eval(_degree_blocks(p, rng)[-1:], 1, 20, min(4, p + 1), 'cpu', rng, 'eval')


def _mixed_blocks(rng, cols):
    """Blocks of different (L, p) (p >= 3, so n_der 4 is valid) with `cols` columns in all: one
    column of L = 48, the others spread over four shorter bases (within 48 KB of coefficients)."""
    shapes = [(48, 8, 'random'), (9, 8, 'uniform'), (20, 5, ('mult', 3)), (13, 3, ('mult', 4)), (16, 4, 'random')]
    ncs = [1] + [len(r) for r in np.array_split(np.arange(cols - 1), 4)]
    blocks, off = [], 0
    for i, ((L, p, kind), nc) in enumerate(zip(shapes, ncs)):
        if nc:
            blocks.append((off, L, nc, p, _knots(kind, p, L, rng, (0., 1.) if i % 2 else (-2.5, 7.))))
            off += L * nc
    return blocks


@pytest.mark.parametrize('cols, n_pts', [(1, 1), (1, 203), (64, 1), (65, 65), (6, 64)])
def test_eval_columns_and_points(emu, cols, n_pts):
    """Blocks of different (L, p) in one call (Lmax strides, the coefficient offsets dsc[5]),
    1, 64 and 65 columns (the 64 threads of omg_eval_kernel stride over columns) and 1, 64, 65 and
    203 points (and over points), n_der 4."""
    rng = np.random.default_rng(cols * 1000 + n_pts)
    blocks = _mixed_blocks(rng, cols) if cols > 1 else [(0, 48, 1, 8, _knots('random', 8, 48, rng))]
    _check_eval(blocks, 2, n_pts, 4, 'cpu', rng, 'eval')


def _eval_args(n_blocks_cols):
    """omg_eval_batch arguments for blocks [(L, p, nc)] with n_der 1 (host buffers)."""
    keep = {}
    offs, lens, ncols, degs, knots, off = [], [], [], [], [], 0
    for L, p, nc in n_blocks_cols:
        offs.append(off); lens.append(L); ncols.append(nc); degs.append(p)
        knots.append(np.r_[np.zeros(p), np.linspace(0, 1, L - p + 1), np.ones(p)])
        off += L * nc
    n = off
    keep['x'] = np.ones((1, n))
    keep['tau'], keep['scale'] = np.array([[0.5]]), np.ones(1)
    keep['out'] = np.zeros(sum(ncols))
    for k, v in (('o', offs), ('l', lens), ('c', ncols), ('p', degs)):
        keep[k] = np.array(v, np.int32)
    keep['k'] = np.concatenate(knots)
    args = [1, n, keep['x'].ctypes.data, len(offs)] + [keep[k].ctypes.data for k in 'olcpk'] + \
        [1, keep['tau'].ctypes.data, keep['scale'].ctypes.data, 1, keep['out'].ctypes.data, None]
    return args, keep


def test_eval_coefficient_limit(emu):
    """Exactly 48 KB of derivative coefficients per instance is accepted and evaluates correctly;
    8 bytes more are rejected with the message."""
    args, keep = _eval_args([(48, 3, 128)])
    assert emu.omg_eval_batch(*args) == 0, emu.omg_last_error()
    assert np.allclose(keep['out'], 1., rtol=0, atol=1e-15)     # partition of unity
    args, keep = _eval_args([(48, 3, 128), (1, 0, 1)])
    assert emu.omg_eval_batch(*args) == -1
    assert emu.omg_last_error().decode() == 'omg_eval_batch: derivative coefficients exceed 48 KB per instance'


# ---------------------------------------------------------------------------------------------
# omg_shift_free_batch
# ---------------------------------------------------------------------------------------------
_SOLVERS = {}


def _solver(n):
    """A problem handle with n variables (only its n matters to the warm start)."""
    key = (n, b200._lib)
    if key not in _SOLVERS:
        _SOLVERS[key] = b200.B200Solver(sk.band(n, 1))
    return _SOLVERS[key]


def _rule(T):
    u, target = (T - DT, T) if T < 2 * DT else (DT, T - DT)
    return u / target, target


def _check_shift_free(blocks, Ts, n, device, rng, family, check=None):
    """Instances b with T = Ts[b] (and a few inactive ones and T outside the rule's range)."""
    slv = _solver(n)
    ti = n - 1
    B = len(Ts) + len(T_OUTSIDE) + 2
    allT = np.r_[Ts, T_OUTSIDE, Ts[:2]]
    X = rng.standard_normal((B, n))
    X[:, ti] = allT
    active = np.ones(B, np.int32)
    active[-2:] = 0
    Xt = _torch(X, device)
    slv.shift_free_batch_device(Xt, blocks, ti, DT, active=_torch(active, device))
    Y = Xt.cpu().numpy()
    for b in range(len(Ts), B):                                  # untouched, bit for bit
        assert np.array_equal(Y[b], X[b]), (family, b)
    check = range(len(Ts)) if check is None else check
    r = 0.
    for b in check:
        tau, target = _rule(Ts[b])
        assert 0. < tau < 1.
        assert Y[b, ti] == target
        for off, L, nc, p, knots in blocks:
            c = X[b, off:off + L * nc].reshape(nc, L).T
            val, _ = se.shift_free(knots, p, c, tau, 1)
            M = se.shift_matrix(knots, p, tau)
            bound = np.array([[4 * (L + p) * se.U * np.abs(c).max() * float(sum(abs(m) for m in M[i]))] * nc
                              for i in range(L)])
            got = Y[b, off:off + L * nc].reshape(nc, L).T
            err = np.array([[float(abs(se.F(got[i, j]) - val[i, j])) for j in range(nc)] for i in range(L)])
            r = max(r, _ratio(family, err, bound))
        assert r <= 1., (family, b, r)
    return Y


def _shift_blocks(p, rng):
    """Degree-p blocks with L at and around the S thresholds and at 48, uniform, random and
    repeated old knots."""
    Ls = sorted({max(p + 1, L) for L in (25, 26, 32, 33, 42, 43, 48)})
    kinds = ['uniform', 'random', ('mult', max(2, p))]
    blocks, off = [], 0
    for i, L in enumerate(Ls):
        nc = 1 + i % 2
        blocks.append((off, L, nc, p, _knots(kinds[i % 3], p, L, rng)))
        off += L * nc
    return blocks, off


@pytest.mark.parametrize('p', range(1, 9))
def test_shift_free_degrees(emu, p):
    """Degrees 1..8, several blocks of different L at and around S = floor(128 / L) thresholds and
    48 in one call, three motion times of the sweep per degree (every value of the sweep over the
    degrees, both branches of the rule)."""
    rng = np.random.default_rng(200 + p)
    blocks, n = _shift_blocks(p, rng)
    Ts = np.array([T_SWEEP[(3 * p + k) % len(T_SWEEP)] for k in range(3)])
    _check_shift_free(blocks, Ts, max(300, n + 1), 'cpu', rng, 'shift_free')
    print('p=%d worst ratio %.3g' % (p, WORST['shift_free']))


def test_shift_free_full_sweep_and_the_opt_in_branch(emu):
    """The whole T sweep on a degree-3 block of 33 and a degree-8 block of 48 with repeated
    knots, on a handle with n = 1250: 8 (n + 2 Lmax + pmax + 1 + 256 + 2 Lmax^2) bytes of shared
    memory, above 48 KB, so the kernel runs only if the call opts in."""
    rng = np.random.default_rng(300)
    blocks = [(0, 33, 2, 3, _knots('random', 3, 33, rng)), (66, 48, 1, 8, _knots(('mult', 5), 8, 48, rng))]
    _check_shift_free(blocks, np.array(T_SWEEP), 1250, 'cpu', rng, 'shift_free')


def test_shift_free_does_not_depend_on_the_thread_schedule(emu, monkeypatch):
    """The elimination has a barrier per pivot: forward, reverse and random fiber orders give
    bit-identical results (degree 8, L = 48 and 43: S = 2 and 2 grid segments)."""
    rng = np.random.default_rng(400)
    blocks = [(0, 48, 1, 8, _knots('random', 8, 48, rng)), (48, 43, 2, 5, _knots(('mult', 3), 5, 43, rng))]
    slv = _solver(300)
    X = rng.standard_normal((3, 300))
    X[:, 299] = [0.7, 1.6, 24.]
    res = {}
    for sched in ('forward', 'reverse', 'random:1'):
        monkeypatch.setenv('OMG_EMU_SCHED', sched)
        Xt = _torch(X, 'cpu')
        slv.shift_free_batch_device(Xt, blocks, 299, DT)
        res[sched] = Xt.numpy().copy()
    assert not np.array_equal(res['forward'], X)
    assert np.array_equal(res['forward'], res['reverse']) and np.array_equal(res['forward'], res['random:1'])


def test_decimal_solve_agrees_with_the_exact_rational_solve():
    """The collocation solve of spline_exact in 120-digit arithmetic equals the Fraction solve to
    far below any bound (degree 5, L = 20 with repeated knots)."""
    rng = np.random.default_rng(500)
    knots = _knots(('mult', 3), 5, 20, rng)
    for tau in (0.01, 0.5):
        Md, Me = se.shift_matrix(knots, 5, tau), se.shift_matrix(knots, 5, tau, exact=True)
        assert max(float(abs(a - b)) for r1, r2 in zip(Md, Me) for a, b in zip(r1, r2)) < 1e-100


# ---------------------------------------------------------------------------------------------
# omg_sample_batch / omg_shift_batch
# ---------------------------------------------------------------------------------------------
def _fixed_case(rng, n, with_T):
    """Blocks [(off, L, nc, S or T)] with L up to 48, ns nc and L nc above 128."""
    from omg_tools_b200.basics.spline import BSplineBasis
    from omg_tools_b200.basics.spline_extra import shiftfirstknot_T, shiftoverknot_T
    blocks, off = [], 0
    for L, p, nc, ns in ((48, 8, 3, 50), (13, 3, 11, 17), (26, 5, 2, 70), (5, 1, 1, 1)):
        knots = _knots('random', p, L, rng)
        if with_T:
            T = shiftoverknot_T(BSplineBasis(knots, p)) if L != 26 else \
                shiftfirstknot_T(BSplineBasis(knots, p), 0.3)
            M = np.asarray(T, dtype=float)
        else:
            pts = _points(knots, ns, rng)
            M = np.array([[float(v) for v in se.basis(knots, p, x)] for x in pts])
        blocks.append((off, L, nc, M))
        off += L * nc
    assert off < n
    return blocks


def _check_fixed(blocks, X, out, kind, family):
    errs, bnds = [], []
    for b in range(X.shape[0]):
        o = 0
        for off, L, nc, M in blocks:
            for c in range(nc):
                col = X[b, off + c * L:off + (c + 1) * L]
                for s in range(M.shape[0]):
                    v, e = se.dot(M[s], col)
                    g = out[b, o + c * M.shape[0] + s] if kind == 'sample' else out[b, off + c * L + s]
                    errs.append(float(abs(se.F(g) - v)))
                    bnds.append(e)
            o += nc * M.shape[0]
    r = _ratio(family, errs, bnds)
    assert r <= 1., (family, r)


def _run_sample(device, n, B, rng):
    blocks = _fixed_case(rng, n, False)
    X = rng.standard_normal((B, n))
    out = b200.sample_batch(_torch(X, device), blocks).cpu().numpy()
    assert out.shape == (B, sum(blk[2] * blk[3].shape[0] for blk in blocks))
    _check_fixed(blocks, X, out, 'sample', 'fixed_rows')


def _run_shift(device, n, B, rng):
    blocks = _fixed_case(rng, n, True)
    X = rng.standard_normal((B, n))
    Xt = _torch(X, device)
    _solver(n).shift_batch_device(Xt, blocks)
    Y = Xt.cpu().numpy()
    _check_fixed(blocks, X, Y, 'shift', 'fixed_rows')
    covered = np.zeros(n, bool)
    for off, L, nc, _ in blocks:
        covered[off:off + L * nc] = True
    assert np.array_equal(Y[:, ~covered], X[:, ~covered])       # outside the blocks: untouched


@pytest.mark.parametrize('n', [400, 7000])
def test_fixed_rows_sample(emu, n):
    """omg_sample_batch: four blocks, exact basis rows (ends, knots, either side, outside) rounded
    to double; n = 400 strides the row load, n = 7000 needs 56 KB of shared memory (opt-in)."""
    _run_sample('cpu', n, 2, np.random.default_rng(600 + n))


def test_fixed_rows_shift(emu):
    """omg_shift_batch: shiftoverknot_T and shiftfirstknot_T matrices, n = 400."""
    _run_shift('cpu', 400, 2, np.random.default_rng(700))


def _fixed_args(emu, kind, h, n, keep):
    x = np.zeros((1, n))
    keep.update(x=x, o=np.array([0, 10], np.int32), l=np.array([5, 4], np.int32), c=np.array([2, 1], np.int32),
                s=np.array([3, 2], np.int32), M=np.ones(5 * 5 + 4 * 4), out=np.zeros(8))
    if kind == 'shift':
        return [h, 1, x.ctypes.data, 2, keep['o'].ctypes.data, keep['l'].ctypes.data, keep['c'].ctypes.data,
                keep['M'].ctypes.data, None]
    return [1, n, x.ctypes.data, 2, keep['o'].ctypes.data, keep['l'].ctypes.data, keep['c'].ctypes.data,
            keep['s'].ctypes.data, keep['M'].ctypes.data, keep['out'].ctypes.data, None]


def test_fixed_rows_bad_arguments_are_rejected(emu):
    """omg_shift_batch / omg_sample_batch: the valid call passes; null pointers, n_blocks < 0,
    len < 1, ncol < 1, nsamp < 1 and blocks outside x are rejected with a message, and so is
    (sample) an x row above 227 KB."""
    slv = _solver(300)
    for kind, fn, idx in (('shift', emu.omg_shift_batch, dict(o=4, l=5, c=6, nb=3, x=2)),
                          ('sample', emu.omg_sample_batch, dict(o=4, l=5, c=6, s=7, nb=3, x=2, out=9))):
        f = 'omg_%s_batch: ' % kind
        keep = {}
        assert fn(*_fixed_args(emu, kind, slv._handle, 300, keep)) == 0, emu.omg_last_error()
        cases = [('x', None, 'null argument'), ('o', None, 'null argument'), ('nb', -1, 'n_blocks -1 < 0'),
                 ('l', [0, 4], 'block 0: basis length 0 < 1'), ('l', [5, -3], 'block 1: basis length -3 < 1'),
                 ('c', [2, 0], 'block 1: columns outside x'), ('o', [-1, 10], 'block 0: columns outside x'),
                 ('o', [0, 297], 'block 1: columns outside x'), ('c', [61, 1], 'block 0: columns outside x')]
        if kind == 'sample':
            cases += [('s', [3, 0], 'block 1: nsamp 0 < 1'), ('out', None, 'null argument')]
        for name, value, message in cases:
            args = _fixed_args(emu, kind, slv._handle, 300, keep)
            if isinstance(value, list):
                keep['bad'] = np.array(value, np.int32)
                args[idx[name]] = keep['bad'].ctypes.data
            else:
                args[idx[name]] = value
            assert fn(*args) == -1, (kind, name, value)
            err = emu.omg_last_error().decode()
            assert err.startswith(f) and message in err, err
    args = _fixed_args(emu, 'sample', None, 227 * 128 + 1, keep)
    assert emu.omg_sample_batch(*args) == -1
    assert emu.omg_last_error().decode() == 'omg_sample_batch: x row exceeds the shared memory of a block'
    args = _fixed_args(emu, 'sample', None, 227 * 128, keep)
    assert emu.omg_sample_batch(*args) == 0, emu.omg_last_error()


def test_wrappers_check_shapes_before_the_call(emu):
    """shift_batch_device: X of the handle's n and T of L x L; sample_batch: S with L columns."""
    slv = _solver(300)
    T = np.eye(5)
    with pytest.raises(ValueError, match='X must be'):
        slv.shift_batch_device(_torch(np.zeros((2, 299)), 'cpu'), [(0, 5, 1, T)])
    with pytest.raises(ValueError, match='5 x 5 T'):
        slv.shift_batch_device(_torch(np.zeros((2, 300)), 'cpu'), [(0, 5, 1, np.eye(4))])
    with pytest.raises(ValueError, match='5 x 5 T'):
        slv.shift_batch_device(_torch(np.zeros((2, 300)), 'cpu'), [(0, 5, 1, np.ones(25))])
    with pytest.raises(ValueError, match='S with 5 columns'):
        b200.sample_batch(_torch(np.zeros((2, 300)), 'cpu'), [(0, 5, 1, np.ones((3, 4)))])
    X = _torch(np.ones((2, 300)), 'cpu')
    slv.shift_batch_device(X, [(0, 5, 1, 2 * T)])
    assert (X[:, :5] == 2).all() and (X[:, 5:] == 1).all()
    assert (b200.sample_batch(X, [(0, 5, 1, np.ones((3, 5)))]) == 10).all()


# ---------------------------------------------------------------------------------------------
# on the device
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_gpu_eval_degrees():
    for p in range(9):
        _run_eval_degree(p, 'cuda', 3)
    print('eval worst ratio %.3g' % WORST['eval'])


@pytest.mark.gpu
@pytest.mark.parametrize('cols, n_pts', [(1, 203), (64, 1), (65, 65), (6, 64)])
def test_gpu_eval_columns_and_points(cols, n_pts):
    rng = np.random.default_rng(cols * 1000 + n_pts)
    blocks = _mixed_blocks(rng, cols) if cols > 1 else [(0, 48, 1, 8, _knots('random', 8, 48, rng))]
    _check_eval(blocks, 2, n_pts, 4, 'cuda', rng, 'eval')


@pytest.mark.gpu
def test_gpu_eval_many_instances():
    """B = 5000, past the resident blocks of 132 SMs (32 blocks of 64 threads each); the first,
    last and a few random instances checked."""
    rng = np.random.default_rng(800)
    blocks = _mixed_blocks(rng, 6)
    _check_eval(blocks, 5000, 30, 4, 'cuda', rng, 'eval', check=np.r_[0, rng.integers(1, 4999, 4), 4999])
    print('eval worst ratio %.3g' % WORST['eval'])


@pytest.mark.gpu
def test_gpu_eval_coefficient_limit():
    import torch
    for extra, ok in (([], True), ([(1, 0, 1)], False)):
        blocks = [(0, 48, 128, 3, np.r_[np.zeros(3), np.linspace(0, 1, 46), np.ones(3)])]
        if extra:
            blocks.append((48 * 128, 1, 1, 0, np.array([0., 1.])))
        X = torch.ones((1, 48 * 128 + 1), dtype=torch.float64, device='cuda')
        tau = torch.full((1, 1), 0.5, dtype=torch.float64, device='cuda')
        if ok:
            out = b200.eval_batch(X, blocks, tau, torch.ones(1, dtype=torch.float64, device='cuda'), 1)
            assert torch.allclose(out, torch.ones_like(out), rtol=0, atol=1e-15)
        else:
            with pytest.raises(RuntimeError, match='derivative coefficients exceed 48 KB per instance'):
                b200.eval_batch(X, blocks, tau, torch.ones(1, dtype=torch.float64, device='cuda'), 1)


@pytest.mark.gpu
@pytest.mark.parametrize('p', range(1, 9))
def test_gpu_shift_free_degrees(p):
    rng = np.random.default_rng(200 + p)
    blocks, n = _shift_blocks(p, rng)
    Ts = np.array([T_SWEEP[(3 * p + k) % len(T_SWEEP)] for k in range(3)])
    _check_shift_free(blocks, Ts, max(300, n + 1), 'cuda', rng, 'shift_free')


@pytest.mark.gpu
def test_gpu_shift_free_full_sweep_and_the_opt_in_branch():
    """n = 1250: above 48 KB of shared memory, the cudaFuncSetAttribute branch."""
    rng = np.random.default_rng(300)
    blocks = [(0, 33, 2, 3, _knots('random', 3, 33, rng)), (66, 48, 1, 8, _knots(('mult', 5), 8, 48, rng))]
    _check_shift_free(blocks, np.array(T_SWEEP), 1250, 'cuda', rng, 'shift_free')
    print('shift_free worst ratio %.3g' % WORST['shift_free'])


@pytest.mark.gpu
@pytest.mark.parametrize('n', [400, 7000])
def test_gpu_fixed_rows_sample(n):
    _run_sample('cuda', n, 3, np.random.default_rng(600 + n))


@pytest.mark.gpu
def test_gpu_fixed_rows_shift():
    _run_shift('cuda', 400, 3, np.random.default_rng(700))
    print('fixed rows worst ratio %.3g' % WORST['fixed_rows'])
