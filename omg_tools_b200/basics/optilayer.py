"""OptiChild / OptiFather: the modelling layer and the drop-in boundary.

Same public interface as the reference's ``omgtools/basics/optilayer.py``
(OptiChild.define_* 556-669, OptiFather.construct_problem 180-198,
get/set_variables 332-380, set_parameters 427-445, update_bounds 313-319,
init_transformations / transform_primal_splines 451-490, create_nlp 49-104),
but without CasADi: symbols are ``Poly`` objects, the composed NLP is lowered
to constant tables (``lowering.lower``) and handed to the B200 solver through
the C-ABI (``solver/b200.py``).  ``create_nlp`` is the exact point where the
reference calls ``nlpsol('solver','ipopt',...)``.
"""
# Attribution: the class / method / option names and the constraint rows of this module restate
# the corresponding module of OMG-tools (omgtools/basics/optilayer.py; Copyright (C) 2016 Ruben Van Parys &
# Tim Mercy, KU Leuven; GNU LGPL v3) -- they are the drop-in contract of this framework.  See NOTICE.
from __future__ import print_function

import collections as col
import copy
import time
from itertools import groupby

import numpy as np

from . import poly as pl
from .poly import Poly
from .spline import BSpline
from .lowering import lower

inf = float('inf')


# ===========================================================================
# flat structs (stand-in for casadi.tools.struct)
# ===========================================================================

class FlatStruct(object):
    """Ordered (label, name) -> column-major block of a flat vector."""

    def __init__(self, entries):
        # entries: list of (label, name, shape)
        self.entries = col.OrderedDict()
        self.labels = col.OrderedDict()
        off = 0
        for label, name, shape in entries:
            size = int(shape[0]) * int(shape[1])
            self.entries[(label, name)] = (off, size, (int(shape[0]), int(shape[1])))
            lo, hi = self.labels.get(label, (off, off))
            self.labels[label] = (min(lo, off), off + size)
            off += size
        self.size = off

    def __call__(self, value=0.):
        return StructVector(self, value)

    def keys(self):
        return list(self.entries.keys())


class StructVector(object):
    """Flat float64 vector with struct indexing, like casadi's DMStruct."""

    def __init__(self, struct, value=0.):
        self.struct = struct
        if isinstance(value, StructVector):
            value = value.cat
        value = np.asarray(value, dtype=float)
        if value.ndim == 0:
            self.cat = np.full(struct.size, float(value))
        else:
            self.cat = value.reshape(-1).astype(float).copy()
            if self.cat.size != struct.size:
                raise ValueError('struct size mismatch: %d vs %d' %
                                 (self.cat.size, struct.size))

    def _locate(self, key):
        if isinstance(key, tuple):
            return self.struct.entries[key]
        if key in self.struct.labels and key is not None:
            lo, hi = self.struct.labels[key]
            return lo, hi - lo, (hi - lo, 1)
        return self.struct.entries[(None, key)]

    def __getitem__(self, key):
        off, size, shape = self._locate(key)
        return self.cat[off:off + size].reshape(shape, order='F')

    def __setitem__(self, key, value):
        off, size, shape = self._locate(key)
        value = np.asarray(value, dtype=float)
        if value.ndim == 0:
            self.cat[off:off + size] = float(value)
            return
        if value.shape == shape:
            self.cat[off:off + size] = value.reshape(-1, order='F')
        elif value.size == size:
            # vectors / lists of columns are taken as given (column-major)
            if value.ndim == 2 and value.shape == (shape[1], shape[0]) and \
                    shape[0] != shape[1]:
                value = value.T
            self.cat[off:off + size] = value.reshape(-1, order='F')
        else:
            raise ValueError('cannot assign shape %s to entry of shape %s' %
                             (value.shape, shape))

    def prefix(self, label):
        return _Prefix(self, label)

    def __array__(self, dtype=None, copy=None):
        return self.cat if dtype is None else self.cat.astype(dtype)

    def __len__(self):
        return self.struct.size


class _Prefix(object):
    def __init__(self, vec, label):
        self.vec, self.label = vec, label

    def __getitem__(self, name):
        return self.vec[(self.label, name)]

    def __setitem__(self, name, value):
        self.vec[(self.label, name)] = value


# ===========================================================================
# solver creation: the reference's L0 crossing
# ===========================================================================

def translate_solver_options(options):
    """Map the reference's option dict to B200-solver options.

    ``options['solver_options']['ipopt']`` keys such as 'ipopt.tol' and
    'ipopt.max_iter' (reference problem.py:54-62) are honoured so existing
    scripts keep working; ``solver_options['b200']`` overrides them.
    """
    out = {}
    so = options.get('solver_options', {})
    for key, value in so.get('ipopt', {}).items():
        if key.startswith('ipopt.'):
            out[key[len('ipopt.'):]] = value
    out.update(so.get('b200', {}))
    return out


def create_nlp(tables, options, name=''):
    """Build the solver object for a lowered NLP (reference optilayer.py:49-104).

    Returns (problem, buildtime); ``problem(x0=, p=, lbg=, ubg=)`` returns a
    dict with 'x', 'lam_g', 'f' and ``problem.stats()['return_status']`` uses
    IPOPT's status strings (reference problem.py:113-128).
    """
    if options.get('verbose', 0) >= 1:
        print('Building nlp ... ', end=' ')
    t0 = time.time()
    solver = options.get('solver', 'b200')
    if solver in ('b200', 'ipopt'):
        # 'ipopt' is accepted as an alias: this framework replaces exactly the
        # CasADi+IPOPT call; there is no CPU fallback.
        from ..solver.b200 import B200Solver
        problem = B200Solver(tables, translate_solver_options(options))
    else:
        raise ValueError('Unknown solver %r (this framework provides "b200")'
                         % solver)
    t1 = time.time()
    if options.get('verbose', 0) >= 1:
        print('in %5f s' % (t1 - t0))
    return problem, (t1 - t0)


# ===========================================================================
# OptiFather
# ===========================================================================

class OptiFather(object):

    def __init__(self, children=None):
        children = children or []
        self.children = col.OrderedDict()
        for child in children:
            self.add(child)

    def add(self, children):
        children = children if isinstance(children, list) else [children]
        for child in children:
            self.children.update({child.label: child})

    # ---------------------------------------------------------------------
    # problem composition
    # ---------------------------------------------------------------------

    def construct_problem(self, options, name='', problem=None):
        self.translate_symbols()
        self.construct_variables()
        self.construct_parameters()
        rows, lb, ub = self.construct_constraints()
        objective = self.construct_objective()
        self.tables = lower(self._var_ids, self._par_ids, rows, objective,
                            lb, ub, self.order_hint())
        self.problem_description = {'tables': self.tables, 'opt': options}
        if problem is None:
            problem, buildtime = create_nlp(self.tables, options, name)
        else:
            buildtime = 0.
        self.init_variables()
        self.init_parameters()
        return problem, buildtime

    def order_hint(self):
        """Relative "time" position of every variable (spline coefficient index /
        basis length): the key of the banded KKT ordering (lowering.py)."""
        hint = np.full(self._var_struct.size, 0.5)
        for (label, name), (off, size, shape) in self._var_struct.entries.items():
            child = self.children[label]
            if name in child._splines_prim and shape[0] > 1:
                L = shape[0]
                for c in range(shape[1]):
                    hint[off + c * L:off + (c + 1) * L] = np.arange(L) / (L - 1.0)
        return hint

    def translate_symbols(self):
        """Resolve named placeholders to the child that defines them
        (reference optilayer.py:204-223)."""
        for label, child in self.children.items():
            for name, symbol in child._symbols.items():
                sym_def = [c for c in self.children.values()
                           if name in c._variables or name in c._parameters]
                if len(sym_def) > 1:
                    raise ValueError('Symbol %s, defined in %s, is defined'
                                     ' multiple times as parameter or'
                                     ' variable by %s!' %
                                     (name, label, ','.join(
                                         [sd.label for sd in sym_def])))
                elif len(sym_def) == 0:
                    raise ValueError('Symbol %s, defined in %s, is not defined'
                                     ' as parameter or variable by any object'
                                     % (name, label))
                owner = sym_def[0]
                target = owner._variables.get(name, None)
                if target is None:
                    target = owner._parameters[name]
                if target.shape != symbol.shape:
                    raise ValueError('Symbol %s of %s has shape %s but %s '
                                     'defines shape %s' % (
                                         name, label, symbol.shape,
                                         owner.label, target.shape))
                for s, t in zip(symbol.reshape(-1), target.reshape(-1)):
                    pl.set_alias(s, t)

    def _flat_ids(self, dictionary_name):
        entries, ids = [], []
        for label, child in self.children.items():
            for name, mat in getattr(child, dictionary_name).items():
                entries.append((label, name, mat.shape))
                ids += [e.single_symbol() for e in mat.reshape(-1, order='F')]
        return FlatStruct(entries), ids

    def construct_variables(self):
        self._var_struct, self._var_ids = self._flat_ids('_variables')

    def construct_parameters(self):
        self._par_struct, self._par_ids = self._flat_ids('_parameters')

    def _expand(self, expr):
        """Substitute the define_substitute placeholders by their expressions."""
        if not self._subst_map:
            return expr
        return pl.substitute(expr, self._subst_map)

    def construct_constraints(self):
        self._subst_map = {}
        for child in self.children.values():
            for name, (expr, subst) in child._substitutes.items():
                for s, e in zip(np.asarray(subst).reshape(-1),
                                np.asarray(expr).reshape(-1)):
                    self._subst_map[s.single_symbol()] = e
        entries, rows, lb, ub = [], [], [], []
        self._constraint_shutdown = {}
        for child in self.children.values():
            for name, constraint in child._constraints.items():
                expr = np.atleast_1d(np.asarray(constraint[0], dtype=object))
                expr = expr.reshape(-1, order='F')
                cname = child._add_label(name)
                entries.append((None, cname, (len(expr), 1)))
                rows += [self._expand(e) for e in expr]
                lb += list(np.broadcast_to(constraint[1], (len(expr),)))
                ub += list(np.broadcast_to(constraint[2], (len(expr),)))
                if constraint[3]:
                    self._constraint_shutdown[cname] = constraint[3]
        self._con_struct = FlatStruct(entries)
        self._lb = self._con_struct(np.array(lb, dtype=float))
        self._ub = self._con_struct(np.array(ub, dtype=float))
        return rows, self._lb.cat, self._ub.cat

    def construct_objective(self):
        objective = Poly()
        for child in self.children.values():
            objective = objective + self._expand(child._objective)
        return objective

    def reset(self):
        for child in self.children.values():
            child.reset()

    # ---------------------------------------------------------------------
    # problem evaluation
    # ---------------------------------------------------------------------

    def update_bounds(self, current_time):
        lb, ub = copy.deepcopy(self._lb), copy.deepcopy(self._ub)
        for name, shutdown in self._constraint_shutdown.items():
            shutdown_fun = eval('lambda t: %s' % shutdown)
            if shutdown_fun(current_time):
                lb[name], ub[name] = -inf, +inf
        return lb, ub

    def init_variables(self):
        variables = self._var_struct(0.)
        for label, child in self.children.items():
            for name in child._variables.keys():
                variables[label, name] = child._values[name]
        self._var_result = variables
        self._dual_var_result = self._con_struct(0.)

    def init_parameters(self):
        self.set_parameters(0.)

    def set_variables(self, variables, child=None, name=None):
        if child is None:
            self._var_result = self._var_struct(variables)
        elif name is None:
            lo, hi = self._var_struct.labels[child.label]
            self._var_result.cat[lo:hi] = np.asarray(variables).reshape(-1)
        else:
            self._var_result[child.label, name] = variables

    def set_dual_variables(self, variables, child=None, name=None):
        if child is None:
            self._dual_var_result = self._con_struct(variables)
        else:
            raise RuntimeError('Error dual variables')

    def _symbol_values(self):
        vals = {}
        for sid, v in zip(self._var_ids, self._var_result.cat):
            vals[pl.resolve(sid)] = float(v)
        for sid, v in zip(self._par_ids, self._par_result.cat):
            vals[pl.resolve(sid)] = float(v)
        return vals

    def _evaluate(self, expr):
        vals = self._symbol_values()
        arr = np.atleast_1d(np.asarray(expr, dtype=object))
        out = np.empty(arr.shape)
        for k, e in enumerate(arr.reshape(-1)):
            e = self._expand(e) if isinstance(e, Poly) else e
            out.reshape(-1)[k] = e.evaluate(vals) if isinstance(e, Poly) \
                else float(e)
        return out

    def get_variables(self, child=None, name=None, **kwargs):
        if child is None:
            return self._var_result
        elif name is None:
            return self._var_result.prefix(child.label)
        want_spline = not ('spline' in kwargs and not kwargs['spline'])
        symbolic = 'symbolic' in kwargs and kwargs['symbolic']
        if name in child._substitutes:
            expr, subst = child._substitutes[name]
            if symbolic:
                coeffs = subst if ('substitute' in kwargs and
                                   not kwargs['substitute']) else expr
            else:
                coeffs = self._evaluate(expr)
            if name in child._splines_prim and want_spline:
                basis = child._splines_prim[name]['basis']
                coeffs = np.asarray(coeffs).reshape(len(basis), -1, order='F')
                return [BSpline(basis, coeffs[:, k])
                        for k in range(coeffs.shape[1])]
            return coeffs
        if symbolic:
            coeffs = child._variables[name]
        else:
            coeffs = np.array(self._var_result[child.label, name])
        if name in child._splines_prim and want_spline:
            basis = child._splines_prim[name]['basis']
            return [BSpline(basis, coeffs[:, k])
                    for k in range(coeffs.shape[1])]
        return coeffs

    def get_dual_variables(self, child=None, name=None, **kwargs):
        if child is None:
            return self._dual_var_result
        raise RuntimeError('Error dual variables')

    def get_parameters(self, child=None, name=None, **kwargs):
        if child is None:
            return self._par_result
        elif name is None:
            return self._par_result.prefix(child.label)
        symbolic = 'symbolic' in kwargs and kwargs['symbolic']
        want_spline = not ('spline' in kwargs and not kwargs['spline'])
        coeffs = child._parameters[name] if symbolic else \
            np.array(self._par_result[child.label, name])
        if name in child._splines_prim and want_spline:
            basis = child._splines_prim[name]['basis']
            return [BSpline(basis, coeffs[:, k])
                    for k in range(coeffs.shape[1])]
        return coeffs

    def get_constraint(self, child, name, symbolic=False):
        expr = self.children[child.label]._constraints[name][0]
        return expr if symbolic else self._evaluate(expr)

    def get_objective(self, child, name=None, symbolic=False):
        expr = self.children[child.label]._objective
        return expr if symbolic else self._evaluate(expr)[0]

    def set_parameters(self, time):
        self._par_result = self._par_struct(0.)
        parameters = {}
        for label, child in self.children.items():
            par = child.set_parameters(time)
            for chld, dic in par.items():
                if chld not in parameters:
                    parameters[chld] = {}
                for key in dic.keys():
                    if key in parameters[chld]:
                        raise ValueError('Same parameter set multiple times!')
                parameters[chld].update(par[chld])
        for label, child in self.children.items():
            for name in child._parameters.keys():
                if child in parameters and name in parameters[child]:
                    self._par_result[label, name] = parameters[child][name]
                else:
                    self._par_result[label, name] = child._values[name]
        return self._par_result

    # ---------------------------------------------------------------------
    # spline transformations (receding-horizon warm start)
    # ---------------------------------------------------------------------

    def init_transformations(self, init_primal_transform, init_dual_transform):
        _init_tf = {}
        for child in self.children.values():
            for name, spl in child._splines_prim.items():
                if name in child._variables or name in child._substitutes:
                    basis = spl['basis']
                    if basis not in _init_tf:
                        _init_tf[basis] = init_primal_transform(basis)
                    child._splines_prim[name]['init'] = _init_tf[basis]
        _init_tf = {}
        for child in self.children.values():
            for name, spl in child._splines_dual.items():
                basis = spl['basis']
                if basis not in _init_tf:
                    _init_tf[basis] = init_dual_transform(basis)
                child._splines_dual[name]['init'] = _init_tf[basis]

    def shifted_entries(self, seg_shift=None):
        """[(offset, len_basis, n_columns, T)] of the spline variables that the
        warm-start knot shift touches: names containing 'seg<k>', k in
        seg_shift (reference optilayer.py:470-490), plus splines a child marks
        with ``_splines_prim[name]['shift'] = True`` (Quadrotor3D's
        acceleration slacks, see vehicles/quadrotor3d.py)."""
        if seg_shift is None:
            seg_shift = [0]
        elif not isinstance(seg_shift, list):
            seg_shift = [seg_shift]
        out = []
        for label, child in self.children.items():
            for name, spl in child._splines_prim.items():
                if name in child._variables:
                    if (('seg' in name and
                            int(name[name.index('seg') + 3]) in seg_shift) or
                            (spl.get('shift') and 0 in seg_shift)):
                        off, size, shape = self._var_struct.entries[(label, name)]
                        out.append((label, name, off, shape, spl.get('init')))
        return out

    def transform_primal_splines(self, transform_fun, seg_shift=None):
        for label, name, off, shape, init in self.shifted_entries(seg_shift):
            basis = self.children[label]._splines_prim[name]['basis']
            if init is not None:
                self._var_result[label, name] = transform_fun(
                    self._var_result[label, name], basis, init)
            else:
                self._var_result[label, name] = transform_fun(
                    self._var_result[label, name], basis)

    def transform_dual_splines(self, transform_fun):
        for label, child in self.children.items():
            for name, spl in child._splines_dual.items():
                basis, init = spl['basis'], spl['init']
                key = child._add_label(name)
                if init is not None:
                    self._dual_var_result[key] = transform_fun(
                        self._dual_var_result[key], basis, init)
                else:
                    self._dual_var_result[key] = transform_fun(
                        self._dual_var_result[key], basis)


# ===========================================================================
# OptiChild
# ===========================================================================

class OptiChild(object):
    _labels = []

    def __init__(self, label):
        self.label = OptiChild._make_label(label)
        self._variables = col.OrderedDict()
        self._parameters = col.OrderedDict()
        self._symbols = col.OrderedDict()
        self._substitutes = col.OrderedDict()
        self._values = col.OrderedDict()
        self._splines_prim = col.OrderedDict()
        self._splines_dual = col.OrderedDict()
        self._constraints = col.OrderedDict()
        self._objective = Poly()
        self._constraint_cnt = 0
        self.n_cons = 0

    def __str__(self):
        return self.label

    __repr__ = __str__

    def _add_label(self, name):
        return name + '_' + self.label

    @classmethod
    def _make_label(cls, label):
        """vehicle -> vehicle0, vehicle1, ... (reference optilayer.py:538-550): the label with the first
        index from its own (0 without one) that no child has taken yet.  The reference finds it by one
        recursive call per taken index; this loop gives the same labels without tying the number of
        children a process may create to the recursion limit."""
        parts = [''.join(g) for _, g in groupby(label, str.isalpha)]
        index, rest = parts[-1], ''.join(parts[:-1])
        if not index.isdigit():
            label, index, rest = label + '0', '0', label
        k = int(index)
        while label in cls._labels:
            k += 1
            label = rest + str(k)
        cls._labels.append(label)
        return label

    # ---------------------------------------------------------------------
    # definition of symbols, variables, parameters, constraints, objective
    # ---------------------------------------------------------------------

    @staticmethod
    def _view(mat):
        """What model code handles: scalar for 1x1, vector for n x 1."""
        if mat.shape == (1, 1):
            return mat[0, 0]
        if mat.shape[1] == 1:
            return mat[:, 0]
        return mat

    def _define(self, name, size0, size1, dictionary, kind, value=None):
        if value is None:
            value = np.zeros((size0, size1))
        # The reference identifies symbols BY NAME when it composes the problem
        # (optilayer.py:204-223, 274-294): an entry defined twice under one name (the
        # obstacle parameters when several vehicles share an environment,
        # environment.py:129; the terminal slacks 'g0', 'g1' of a multi-vehicle
        # point-to-point problem, point2point.py:160-163) is ONE entry of the
        # variable / parameter vector.  Symbols here are identified by id, so the
        # first definition is reused.
        if name in dictionary and dictionary[name].shape == (size0, size1):
            self._values[name] = value
            return dictionary[name]
        dictionary[name] = pl.sym_array(self._add_label(name), kind,
                                        size0, size1)
        self._values[name] = value
        return dictionary[name]

    def define_symbol(self, name, size0=1, size1=1):
        # a child may ask for the same placeholder several times (Quadrotor3D
        # takes 't' in init() and again in the collision constraints): all of
        # them must resolve, so the first definition is reused
        if name in self._symbols and self._symbols[name].shape == (size0, size1):
            return self._view(self._symbols[name])
        return self._view(self._define(name, size0, size1, self._symbols, 'sym'))

    def define_variable(self, name, size0=1, size1=1, **kwargs):
        return self._view(self._define(name, size0, size1, self._variables,
                                       'var', kwargs.get('value')))

    def define_parameter(self, name, size0=1, size1=1, **kwargs):
        return self._view(self._define(name, size0, size1, self._parameters,
                                       'par', kwargs.get('value')))

    def _define_spline(self, name, size0, size1, dictionary, kind, basis, value):
        if size1 > 1:
            return [self._define_spline(name + str(l), size0, 1, dictionary,
                                        kind, basis, value)
                    for l in range(size1)]
        coeffs = self._define(name, len(basis), size0, dictionary, kind, value)
        self._splines_prim[name] = {'basis': basis}
        return [BSpline(basis, coeffs[:, k]) for k in range(size0)]

    def define_spline_symbol(self, name, size0=1, size1=1, **kwargs):
        return self._define_spline(name, size0, size1, self._symbols, 'sym',
                                   kwargs.get('basis', getattr(self, 'basis', None)),
                                   kwargs.get('value'))

    def define_spline_variable(self, name, size0=1, size1=1, **kwargs):
        return self._define_spline(name, size0, size1, self._variables, 'var',
                                   kwargs.get('basis', getattr(self, 'basis', None)),
                                   kwargs.get('value'))

    def define_spline_parameter(self, name, size0=1, size1=1, **kwargs):
        return self._define_spline(name, size0, size1, self._parameters, 'par',
                                   kwargs.get('basis', getattr(self, 'basis', None)),
                                   kwargs.get('value'))

    def define_substitute(self, name, expr):
        """Name an expression; constraints written in terms of the returned
        placeholder are expanded at composition (reference optilayer.py:579-605)."""
        if isinstance(expr, list):
            return [self.define_substitute(name + str(l), e)
                    for l, e in enumerate(expr)]
        if name in self._substitutes:
            raise ValueError('Name %s already used for substitutes!' % (name))
        symbol_name = self._add_label(name)
        if isinstance(expr, BSpline):
            self._splines_prim[name] = {'basis': expr.basis}
            coeffs = pl.sym_array(symbol_name, 'sym', len(expr.coeffs), 1)[:, 0]
            self._substitutes[name] = [expr.coeffs, coeffs]
            return BSpline(expr.basis, coeffs)
        arr = np.atleast_1d(np.asarray(expr, dtype=object))
        subst = pl.sym_array(symbol_name, 'sym', arr.size, 1)[:, 0]
        self._substitutes[name] = [arr.reshape(-1), subst]
        return subst if arr.size > 1 else subst[0]

    def set_value(self, name, value):
        self._values[name] = value

    def define_constraint(self, expr, lb, ub, shutdown=False, name=None, skip=[]):
        if isinstance(expr, (float, int)):
            return
        if name is None:
            name = 'c_' + str(self._constraint_cnt)
        else:
            name = name + '_' + str(self._constraint_cnt)
        self._constraint_cnt += 1
        if shutdown and np.all(np.asarray(lb) == np.asarray(ub)):
            # the equality rows are part of the KKT STRUCTURE the solver factorises (the border
            # of the condensed system): they cannot be switched off by the bounds at run time
            # the way an inequality row can.  (No model of the reference does this.)
            raise NotImplementedError(
                "define_constraint(..., shutdown=%r) on an equality constraint (lb == ub) is not "
                "supported by the 'b200' solver: shut down an inequality pair lb <= expr <= ub "
                "instead, or build two problems" % (shutdown,))
        if isinstance(expr, BSpline):
            coeffs = expr.coeffs
            if skip:
                stop = len(coeffs) - skip[1]
                coeffs = coeffs[skip[0]:stop]
            self._constraints[name] = (
                coeffs, lb * np.ones(len(coeffs)), ub * np.ones(len(coeffs)),
                shutdown)
            self._splines_dual[name] = {'basis': expr.basis}
        else:
            self._constraints[name] = (expr, lb, ub, shutdown)
        self.n_cons += np.atleast_1d(
            np.asarray(self._constraints[name][0], dtype=object)).size

    def define_objective(self, expr):
        if isinstance(expr, np.ndarray):
            expr = expr.reshape(-1)[0]
        self._objective = self._objective + expr

    # ---------------------------------------------------------------------
    # reset
    # ---------------------------------------------------------------------

    def reset(self):
        self._variables = col.OrderedDict()
        self._parameters = col.OrderedDict()
        self._symbols = col.OrderedDict()
        self._substitutes = col.OrderedDict()
        self._values = col.OrderedDict()
        self._splines_prim = col.OrderedDict()
        self._splines_dual = col.OrderedDict()
        self._constraints = col.OrderedDict()
        self._objective = Poly()
        self._constraint_cnt = 0

    # ---------------------------------------------------------------------
    # methods required to override
    # ---------------------------------------------------------------------

    def set_parameters(self, time):
        return {}
