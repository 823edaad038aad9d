/* omg_b200.h -- C ABI of libomgb200.so: batched spline-NLP interior-point solve
 * on NVIDIA H100 (sm_90a).
 *
 * This library replaces, for OMG-tools' per-MPC-step solve, the CasADi+IPOPT
 * call of the reference:
 *
 *   omg_problem_create   <->  nlpsol('solver','ipopt',{x,p,f,g},opts)
 *                              omgtools/basics/optilayer.py:49-60 (create_nlp);
 *                              C++ twin: Point2Point.cpp:80-91 (nlpsol(..."nlp.so"))
 *   omg_solve_batch      <->  result = self.problem(x0=var,p=par,lbg=lb,ubg=ub)
 *                              omgtools/problems/problem.py:113 (and admm.py:390);
 *                              C++ twin: Point2Point::solve, Point2Point.cpp:207-231
 *   status/iters arrays  <->  self.problem.stats()['return_status']
 *                              omgtools/problems/problem.py:119-128
 *   omg_feas_batch       <->  (IPOPT's restoration phase inside the same nlpsol call)
 *   omg_shift_batch      <->  father.transform_primal_splines(T.dot(coeffs))
 *                              omgtools/problems/point2point.py:187-198,
 *                              optilayer.py:470-490; C++: transformSplines,
 *                              export.py:406-444
 *   omg_problem_destroy  <->  (garbage collection of the casadi Function)
 *
 * Conventions: plain C, no C++/torch types.  Unless a function name ends in
 * _host, all data pointers are DEVICE pointers owned by the caller; the library
 * owns only the uploaded tables and its workspaces.  Calls on one handle are
 * stream-ordered and not re-entrant.  Every function returns 0 on success or a
 * negative error code; omg_last_error() gives the message (thread-local).
 * Nothing throws across this boundary.
 */
#ifndef OMG_B200_H
#define OMG_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define OMG_ABI_VERSION 6

/* CSR list of polynomial terms per output slot:
 *   out[s] = sum_{t in [ptr[s],ptr[s+1])} coef[t] * V[cidx[t]]
 *            * prod_{k<width} x_ext[xi[t*width+k]]   ( * lam_ext[lrow[t]] if lrow )
 * x_ext = [x, 1, mids], lam_ext = [lambda (m rows), obj_factor, mu (n_mid)].
 *
 * Intermediates ("mids", n_mid >= 0): polynomials of x shared by many rows (the
 * graph nodes CasADi shares in the reference's expression graph; Quadrotor3D's
 * acceleration product splines, quadrotor3d.py:91-126).  They are the outputs
 * m .. m+n_mid-1 of G; rows are affine in them.  The J term list then has
 * nnz_jx >= nnz_j slots: [0,nnz_j) the constraint Jacobian (direct part),
 * then A = d row/d mid, then C = d mid/d x, and
 *     J[s] += sum_{e in [jp_ptr[s],jp_ptr[s+1])} Jx[jp_a[e]] * Jx[jp_c[e]]
 *     mu_l  = sum_{e in [mu_ptr[l],mu_ptr[l+1])} lambda[mu_row[e]] * Jx[mu_slot[e]]
 * give the chain rule for the Jacobian and the multipliers of the mids' own
 * Hessians (W terms with lrow = m+1+l).  The coefficient of a mid in a row may
 * depend on x (a hyperplane normal times an integrated position: Dubins, AGV, trailer;
 * dubins.py:235-251) or on another mid (the steering-rate rows of the bicycle,
 * bicycle.py:115-124): the A slots are then functions of x_ext and the W term list
 * carries nnz_wx extra slots after its nnz_w regular ones, with values Wx:
 *     X[l,k]   = sum_i lambda_i d2 row_i / d mid_l d x_k       (cross slots)
 *     M[l1,l2] = sum_i lambda_i d2 row_i / d mid_l1 d mid_l2   (l1 >= l2)
 * Their contribution X^T C + C^T X + C^T M C to the Hessian is gathered per H position:
 *     H[xq_h[e]] += sum_{r in [xq_ptr[e],xq_ptr[e+1])} Wx[xq_w[r]] * Jx[xq_a[r]] * Jx[xq_b[r]]
 * where xq_b[r] = -1 stands for a factor 1 (cross terms; listed twice on the diagonal). */
typedef struct omg_termlist {
  int32_t n_out, n_terms, width;
  const int32_t* ptr;   /* [n_out+1] */
  const double*  coef;  /* [n_terms] */
  const int32_t* cidx;  /* [n_terms] index into the parameter tape V */
  const int32_t* xi;    /* [n_terms*width] indices into x_ext (n = constant 1) */
  const int32_t* lrow;  /* [n_terms] or NULL */
} omg_termlist;

/* Lowered NLP  min f(x,p)  s.t.  lbg <= g(x,p) <= ubg  (HOST pointers; copied
 * by omg_problem_create).  Built by omg_tools_b200/basics/lowering.py. */
typedef struct omg_tables {
  int32_t abi_version;
  int32_t n, m, n_par, n_v, degree;
  /* parameter tape: V[0]=1, V[1..n_par]=p, entry e -> V[1+n_par+e] =
   * func( sum_t coef[t]*V[f0]*V[f1]*V[f2]*V[f3] ), evaluated level by level */
  int32_t n_tape, n_tape_terms, n_levels;
  const int32_t* tape_func;   /* [n_tape] 0 id,1 inv,2 ge0,3 gt0,4 sin,5 cos,6 sqrt */
  const int32_t* tape_ptr;    /* [n_tape+1] */
  const double*  tape_coef;   /* [n_tape_terms] */
  const int32_t* tape_fac;    /* [n_tape_terms*4] */
  const int32_t* level_ptr;   /* [n_levels+1] entry ranges per level */
  omg_termlist G, F, DF, J, W;
  /* Jacobian pattern, slots sorted by (row, col) */
  int32_t nnz_j;
  const int32_t* jrow; const int32_t* jcol; const int32_t* jrow_ptr; /* [m+1] */
  /* intermediates (see omg_termlist); n_mid = 0: all of this is unused */
  int32_t n_mid, nnz_jx, n_jp, n_mu;
  const int32_t* jp_ptr; const int32_t* jp_a; const int32_t* jp_c;   /* [nnz_j+1],[n_jp] */
  const int32_t* mu_ptr; const int32_t* mu_row; const int32_t* mu_slot; /* [n_mid+1],[n_mu] */
  /* Lagrangian-Hessian pattern (lower triangle) and its position in H */
  int32_t nnz_w;
  const int32_t* wrow; const int32_t* wcol; const int32_t* w2h;
  /* condensed KKT pattern H = W + J^T Sigma J: gather lists of slot pairs */
  int32_t nnz_h, n_hp;
  const int32_t* hrow; const int32_t* hcol; const int32_t* hp_ptr; /* [nnz_h+1] */
  const int32_t* hp_s1; const int32_t* hp_s2; const int32_t* hp_row; /* [n_hp] */
  /* default bounds: rows with lbg==ubg are the structural equality rows */
  const double* lbg; const double* ubg;
  /* condensed KKT K = [[H,Jc^T],[Jc,-dc I]] = L S L^T: fill-reducing symmetric
   * permutation, signs S, lower envelope (row i stored from env_first[i], a
   * multiple of 8, to i; row kkt_n = right-hand side) and the rows reached by
   * each 8-column panel (lowering.build_kkt_structure) */
  int32_t kkt_n, kkt_n_eq, env_size, n_panel_rows, max_panel_rows;
  const int32_t* kkt_eq_rows;   /* [kkt_n_eq] constraint rows that are equalities */
  const int32_t* kkt_pos_var;   /* [n] permuted index of variable j */
  const int32_t* kkt_pos_eq;    /* [kkt_n_eq] permuted index of equality row k */
  const int32_t* kkt_sign;      /* [kkt_n] +1 / -1 */
  const int32_t* env_first;     /* [kkt_n+1] */
  const int32_t* env_ptr;       /* [kkt_n+2] */
  const int32_t* kkt_hdst;      /* [nnz_h] envelope offset of H position q */
  const int32_t* kkt_jdst;      /* [nnz_j] envelope offset of J slot (eq rows) or -1 */
  const int32_t* kkt_diag;      /* [kkt_n] envelope offset of the diagonal */
  const int32_t* kkt_panel_ptr; /* [n_panels+1] */
  const int32_t* kkt_panel_rows;/* [n_panel_rows] */
  /* extra Hessian products (see omg_termlist); nnz_wx = 0: unused.  W.n_out = nnz_w + nnz_wx */
  int32_t nnz_wx, n_xq, n_xp;
  const int32_t* xq_h;          /* [n_xq] H position */
  const int32_t* xq_ptr;        /* [n_xq+1] */
  const int32_t* xq_w;          /* [n_xp] extra W slot (0-based within the extra slots) */
  const int32_t* xq_a;          /* [n_xp] J slot of C = d mid / d x */
  const int32_t* xq_b;          /* [n_xp] second J slot of C, or -1 */
} omg_tables;

/* Interior-point options; defaults = the reference's IPOPT settings
 * (problem.py:57-60) + IPOPT defaults.  Fill with omg_default_options first. */
typedef struct omg_options {
  double tol, constr_viol_tol, dual_inf_tol, compl_inf_tol;
  double mu_init, bound_push, bound_frac, mult_bound_push, bound_relax_factor;
  double scaling_max_gradient;
  int32_t max_iter;
  int32_t trace;          /* 1: record per-iteration diagnostics (debug) */
  /* feasibility restart, the stand-in for IPOPT's restoration phase: when the
   * filter line search fails, keep x, re-centre the slacks (push restart_push),
   * zero the multipliers, clear the filter and continue from mu = restart_mu;
   * at most max_restarts times, then Restoration_Failed. */
  int32_t max_restarts;
  int32_t soft_resto;     /* 1: IPOPT's soft restoration -- when the filter rejects every trial step,
                           * accept the step if it reduces the primal-dual error by 1e-4 (default 1) */
  double restart_mu, restart_push;
  /* inertia test of the factorisation K = L S L^T.  0 (default): IPOPT's -- S takes the
   * sign of every pivot as it comes and the step is accepted when the NUMBER of negative
   * pivots equals the number of equality rows (Sylvester); 1: the stricter positional
   * test (variables +, equality rows -) of the first kernel versions, which over-
   * regularises problems with non-convex constraints. */
  int32_t inertia_mode;
  int32_t reserved;
} omg_options;

/* per-instance status codes (mapped to IPOPT strings in solver/b200.py) */
enum {
  OMG_SOLVE_SUCCEEDED = 0,
  OMG_MAX_ITER_EXCEEDED = 1,
  OMG_RESTORATION_FAILED = 2,
  OMG_ERROR_IN_STEP_COMPUTATION = 3,
  OMG_INVALID_NUMBER_DETECTED = 4,
  OMG_INFEASIBLE_PROBLEM_DETECTED = 5
};

typedef struct omg_problem omg_problem;   /* opaque handle */

void omg_default_options(omg_options* opt);

/* Upload tables to `device`, size workspaces.  Returns NULL on error. */
omg_problem* omg_problem_create(const omg_tables* tables,
                                const omg_options* opt, int device);
void omg_problem_destroy(omg_problem* h);
int  omg_set_options(omg_problem* h, const omg_options* opt);

/* Solve B independent instances of the structure (DEVICE pointers, row-major
 * [B][.] ; lbg/ubg are [m] if bounds_shared else [B][m]; lam_g0 may be NULL).
 * stream: a cudaStream_t (NULL = default stream).  Asynchronous. */
int omg_solve_batch(omg_problem* h, int32_t B,
                    const double* x0, const double* p,
                    const double* lbg, const double* ubg, int32_t bounds_shared,
                    const double* lam_g0,
                    double* x, double* lam_g, double* f,
                    int32_t* status, int32_t* iters, void* stream);

/* omg_solve_batch on the rows listed in DEVICE rows [*n_rows] (n_rows a DEVICE int32): listed
 * entry i solves row rows[i] of every buffer; an unlisted row's outputs are not written.  The
 * launch shape depends on B only, so the list may change between replays of a CUDA graph. */
int omg_solve_batch_rows(omg_problem* h, int32_t B,
                         const double* x0, const double* p,
                         const double* lbg, const double* ubg, int32_t bounds_shared,
                         const double* lam_g0,
                         double* x, double* lam_g, double* f,
                         int32_t* status, int32_t* iters,
                         const int32_t* rows, const int32_t* n_rows, void* stream);

/* Same call with HOST buffers: H2D of inputs, solve, D2H of results,
 * synchronous.  This is the call the reference-facing plugin times end to end. */
int omg_solve_batch_host(omg_problem* h, int32_t B,
                         const double* x0, const double* p,
                         const double* lbg, const double* ubg,
                         int32_t bounds_shared, const double* lam_g0,
                         double* x, double* lam_g, double* f,
                         int32_t* status, int32_t* iters);

/* Feasibility phase, the fallback the host runs on instances that came back with
 * OMG_RESTORATION_FAILED before solving them once more (stand-in for the feasibility
 * part of IPOPT's restoration phase, which the reference relies on implicitly through
 * nlpsol(...,'ipopt',...), optilayer.py:55-60 / problem.py:113-128): up to max_steps
 * Levenberg-Marquardt steps on the violation v(x) = g(x,p) - clip(g(x,p), lbg, ubg),
 * (Jv^T Jv + lam I) dx = -Jv^T v, lam from 1e-3, /10 on an accepted step, x10 (at most
 * 12 times) on a rejected one; stops when max|v| <= 1e-8.  DEVICE pointers; x [B][n],
 * viol [B] (max |v| at the returned point), steps [B].  Asynchronous on `stream`. */
int omg_feas_batch(omg_problem* h, int32_t B,
                   const double* x0, const double* p,
                   const double* lbg, const double* ubg, int32_t bounds_shared,
                   int32_t max_steps, double* x, double* viol, int32_t* steps,
                   void* stream);
/* Same call with HOST buffers (synchronous). */
int omg_feas_batch_host(omg_problem* h, int32_t B,
                        const double* x0, const double* p,
                        const double* lbg, const double* ubg, int32_t bounds_shared,
                        int32_t max_steps, double* x, double* viol, int32_t* steps);

/* Receding-horizon warm start: x[b, off:off+len*ncol] <- T (len x len) applied
 * to each of the ncol columns, for n_blocks spline variables (DEVICE x,
 * in place).  offs/lens/ncols: HOST int arrays [n_blocks]; T: HOST array of the
 * n_blocks row-major matrices, concatenated.  Asynchronous on `stream`; the block
 * descriptor is uploaded on the first call and whenever it changes (the host arrays are
 * copied before the call returns).  The x row is staged in shared memory: 8 n bytes, opted in
 * above 48 KB, up to 227 KB.  Rejected with a message: null pointers, n_blocks < 0, a block with
 * len < 1 or ncol < 1 or outside x (off < 0 or off + len * ncol > n), and n above 227 KB of x row. */
int omg_shift_batch(omg_problem* h, int32_t B, double* x,
                    int32_t n_blocks, const int32_t* offs, const int32_t* lens,
                    const int32_t* ncols, const double* T, void* stream);

/* Debug trace of the last omg_solve_batch with opt.trace=1: per iteration of
 * instance 0, 8 doubles {iter, f, constr_inf, dual_inf, mu, E0, alpha, delta_w}.
 * Copies up to max_rows rows to HOST `out`; returns the number of rows. */
int omg_get_trace(omg_problem* h, double* out, int32_t max_rows);

/* Introspection */
int omg_get_info(omg_problem* h, int32_t* n, int32_t* m, int32_t* n_par,
                 int32_t* smem_bytes, int32_t* ctas_per_sm, int32_t* n_sm);
/* Which kernel family serves this problem and its structure, as one line of text (e.g.
 * "sparse LDL^T: N=200 nnz(L)=3861 levels=29 root=36 pairs=41088 nt=128 ctas/SM=4 smem=53104"
 * or "envelope kernels (intermediates)").  Valid until the handle is destroyed. */
const char* omg_structure_info(omg_problem* h);
/* Layout of the envelope kernels for this problem (the kernels of inertia_mode = 1 and of what
 * the sparse kernel does not take): "kernel=<standard|xl> nt=<threads per block>
 * K=<shared|scratch> V=<shared|scratch> arrays-in-scratch=<per-instance arrays in scratch>
 * max-panel-rows=.. min-panel-rows=.. N%8=.. wide=<0|1>" -- where the KKT envelope K and the
 * parameter tape V live, the most and fewest rows a panel of the factorisation reaches (the
 * last panel, which reaches only the right-hand side, left out of the fewest), and whether
 * panels reach more rows than a block has threads.  Valid until the handle is destroyed. */
const char* omg_envelope_layout(omg_problem* h);
/* Device time (ms) and kernel-launch count of the last omg_solve_batch,
 * measured with CUDA events on the caller's stream. */
int omg_last_timing(omg_problem* h, float* kernel_ms, int32_t* launches);

/* Batched spline sampling (post-solve trajectory extraction, reference
 * Vehicle.store -> sample_splines, omgtools/vehicles/vehicle.py:250-300,
 * spline_extra.py:406-410; C++ twin Vehicle.cpp:112-190): for each of n_blocks
 * spline variables (offset, basis length, columns) apply the HOST matrix
 * S_blk [nsamp x len] (precomputed basis / derivative rows) to every column:
 * out[b] = concat_blk( [col][sample] ), DEVICE x [B][n] and out [B][sum nsamp*ncols].
 * Asynchronous on `stream`; descriptor and S are uploaded on the first call of the host
 * thread and whenever they change (copied before the call returns).  The x row is staged in
 * shared memory as by omg_shift_batch (8 n bytes, up to 227 KB).  Rejected with a message: null
 * pointers, n_blocks < 0, a block with len < 1, ncol < 1 or nsamp < 1 or outside x, and n above
 * 227 KB of x row. */
int omg_sample_batch(int32_t B, int32_t n, const double* x, int32_t n_blocks,
                     const int32_t* offs, const int32_t* lens, const int32_t* ncols,
                     const int32_t* nsamp, const double* S, double* out, void* stream);

/* Per-instance spline bases (free motion time, where every instance has its own T and so its own
 * abscissae).  The spline variables are given as n_blocks blocks (HOST int arrays offs, lens, ncols,
 * degrees [n_blocks]: offset in x, basis length L, columns, degree p; HOST knots: the L + p + 1
 * knots of each block, concatenated), column c of block k at x[b, offs[k] + c * L ..].  Bounds of
 * both calls: 0 <= p <= OMG_SPL_MAX_DEGREE and p + 1 <= L <= OMG_SPL_MAX_LEN.  Basis values follow
 * BSplineBasis.eval_basis (reference spline.py:131-136, 214-233): Cox-de Boor, the leading clamped
 * intervals closed on both ends, every other interval (k_i, k_i+1], zero-length spans skipped.
 * Descriptors are uploaded by the call, which copies the host arrays before it returns.
 * Asynchronous on `stream`. */
#define OMG_SPL_MAX_DEGREE 8
#define OMG_SPL_MAX_LEN 48

/* Free-T warm start, the per-instance counterpart of omg_shift_batch (reference
 * FreeTPoint2point.init_step, point2point.py:354-368, with shift_spline, spline_extra.py:88-99,
 * and BSplineBasis.transform, spline.py:280-306).  For every instance b with active[b] != 0
 * (active: DEVICE int32 [B], or NULL for all): T = x[b, t_index]; u = T - update_time and
 * target = T if T < 2 update_time, else u = update_time and target = T - update_time;
 * tau = u / target.  Each block is re-expressed on the basis with knots [tau] * p +
 * linspace(tau, end, L - p + 1) + [end] * p (end: the block's last knot), collocated at the first
 * arg-max of each new basis function over linspace(tau, end, 501); the transformation's entries
 * below 1e-10 are dropped.  Then x[b, t_index] = target.  Instances with tau outside (0, 1) are
 * left alone.  x: DEVICE [B][n] with n the problem's, in place.  Rejected with a message:
 * update_time <= 0, t_index outside [0, n), null pointers, blocks outside x, and degrees or
 * lengths beyond the bounds above. */
int omg_shift_free_batch(omg_problem* h, int32_t B, double* x, int32_t t_index, double update_time,
                         const int32_t* active, int32_t n_blocks, const int32_t* offs,
                         const int32_t* lens, const int32_t* ncols, const int32_t* degrees,
                         const double* knots, void* stream);

/* Per-instance spline evaluation, the counterpart of omg_sample_batch for abscissae that differ
 * between instances (reference Vehicle.store -> splines2signals at t / T, vehicle.py:250-300):
 * out[b] = concat over blocks of [column][point][derivative], the d-th derivative (d < n_der) of
 * the column at tau[b][j] divided by scale[b]^d.  Derivatives as BSplineBasis.derivative
 * (spline.py:236-260).  DEVICE x [B][n], tau [B][n_pts], scale [B], out
 * [B][sum ncols * n_pts * n_der].  Any finite tau is valid (outside the knot span every value is
 * 0): callers pad their point sets with such points.  Rejected with a message: n_der outside
 * 1 .. 4 or above p + 1 of a block, n_pts < 1, null pointers, blocks outside x, degrees or lengths
 * beyond the bounds above, and more than 48 KB of derivative coefficients per instance. */
int omg_eval_batch(int32_t B, int32_t n, const double* x, int32_t n_blocks, const int32_t* offs,
                   const int32_t* lens, const int32_t* ncols, const int32_t* degrees,
                   const double* knots, int32_t n_pts, const double* tau, const double* scale,
                   int32_t n_der, double* out, void* stream);

/* Non-ideal state prediction for a batch (DEVICE pointers): integrate the vehicle ODE from
 * state0 [B x n_state] over `steps` samples of the planned input trajectory
 * inputs [B x (steps+1) x n_input] with classical RK4, result in stateT [B x n_state].
 * Reference: Vehicle.predict / integrate_ode (vehicle.py:302-337, 412-423), C++ twin
 * Vehicle::predict / integrate (export/vehicles/Vehicle.cpp:61-110; stages 1-3 use
 * input[i], stage 4 input[i+1]).  Unlike the C++ twin, which evaluates every step's
 * stages at the initial state, the running state is used (identical for the holonomic
 * integrator model).  model: 0 integrator (state' = input: Holonomic, Holonomic1D/3D),
 * 1 Quadrotor3D (8 states, 3 inputs; quadrotor3d.py:308-312), 2 planar Quadrotor
 * (5 states, 2 inputs; quadrotor.py:154-157), 3 Dubins (3 states, 2 inputs: x' = v cos theta,
 * y' = v sin theta, theta' = omega), 4 HolonomicOrient (integrator, 3 states and inputs),
 * 5 SimpleQuadrotor3D (Quadrotor3D's 8 states, 3 inputs and ODE). */
int omg_integrate_rk4(int32_t model, int32_t B, int32_t n_state, int32_t n_input,
                      const double* state0, const double* inputs, double sample_time,
                      int32_t steps, double* stateT, void* stream);

/* Closed-loop plant step of a batch after the solve of MPC step `step` (reference
 * Vehicle.simulate / predict with ideal_update = ideal_prediction = False, vehicle.py:302-337,
 * 359-449).  DEVICE: x [B x n] spline coefficients (column c of the input splines at c*L),
 * plant_x [B x n_state], plant_u [B x n_input] (plant state and last applied input at t_k),
 * outputs plant_x_next, plant_u_next (at t_k + n_samp*sample_time; may alias plant_x,
 * plant_u), pred_x, pred_u, and scratch [B x n_input x (n_traj + 24)] (disturb only).
 * HOST: R0, R1 [(n_samp+1) x L] basis and derivative rows (derivative divided by the horizon
 * time) at the samples t_k + s*sample_time; filt = {b[4], a[4], lfilter_zi[3]} of
 * butter(3, fc); mean, stdev [n_input].  Both halves integrate with classical RK4 on the
 * linearly interpolated input (u_i; (u_i+u_i+1)/2 at both midpoints; u_i+1):
 *   simulate: planned input + disturbance (white noise, Philox4x32-10 keyed by seed and
 *             (step, instance, signal, sample), Box-Muller, filtfilt over n_traj samples)
 *             -> first-order lag u' = (u_cmd - u)/time_constant from plant_u (lag != 0)
 *             -> vehicle ODE from plant_x: plant_x_next, plant_u_next = last input sample
 *   predict:  planned input -> vehicle ODE from plant_x: pred_x, pred_u = planned input at
 *             sample n_samp.
 * model: 0 integrator (Holonomic, Holonomic3D; input = ds/dt), 1 Quadrotor3D (thrust and
 * angular rates from f~, q_phi, q_theta).  Rejected: other models, n_traj <= 12 with the
 * disturbance (filtfilt's padding), time_constant <= 0 with the lag, null pointers. */
int omg_closed_loop_step(int32_t model, int32_t B, int32_t n_state, int32_t n_input, int32_t n,
                         const double* x, int32_t L, int32_t n_samp, const double* R0,
                         const double* R1, double sample_time, int32_t lag, double time_constant,
                         int32_t disturb, int32_t n_traj, const double* filt, const double* mean,
                         const double* stdev, uint64_t seed, int32_t step, const double* plant_x,
                         const double* plant_u, double* plant_x_next, double* plant_u_next,
                         double* pred_x, double* pred_u, double* scratch, void* stream);

/* omg_closed_loop_step for every vehicle model with a planned-input map, the ones that need
 * higher derivatives of the flat outputs included.  The derivative rows come as ONE host array
 * R [n_der x (n_samp+1) x L]: row d is the d-th derivative of the basis divided by T^d at the
 * samples t_k + s*sample_time (n_der from 2 to 4: value, first, second, third derivative).
 * Every other argument, the outputs and the integration are omg_closed_loop_step's, which
 * forwards here with n_der = 2 (results bit-identical).  Models and the planned input they
 * take from the spline columns (the vehicle's splines2signals; g = 9.81), n_state / n_input,
 * the n_der they need, and the ODE:
 *   0 integrator  (Holonomic, Holonomic3D)  n / n  2  input = ds/dt; s' = input
 *   1 Quadrotor3D  8 / 3  2  thrust and angular rates from f~, q_phi, q_theta
 *   2 Quadrotor    5 / 2  4  u1 = sqrt(x''^2 + (y''+g)^2),
 *                            u2 = (x'''(y''+g) - x'' y''') / ((y''+g)^2 + x''^2); quadrotor.py ode
 *   3 Dubins       3 / 2  2  v = v~ (1 + tg^2), omega = 2 tg' / (1 + tg^2);
 *                            (v cos theta, v sin theta, omega)
 *   4 HolonomicOrient 3 / 3  2  (x', y', 2 tg' / (1 + tg^2)); integrator
 *   5 SimpleQuadrotor3D 8 / 3  4  u1, u2, u3 of quadrotor3d_simple.py (az = z'' + g);
 *                            Quadrotor3D's ODE
 * Rejected with a message: unknown models, sizes that do not match the model, n_der below the
 * model's or above 4, and everything omg_closed_loop_step rejects. */
int omg_closed_loop_step_der(int32_t model, int32_t B, int32_t n_state, int32_t n_input, int32_t n,
                             const double* x, int32_t L, int32_t n_samp, int32_t n_der,
                             const double* R, double sample_time, int32_t lag,
                             double time_constant, int32_t disturb, int32_t n_traj,
                             const double* filt, const double* mean, const double* stdev,
                             uint64_t seed, int32_t step, const double* plant_x,
                             const double* plant_u, double* plant_x_next, double* plant_u_next,
                             double* pred_x, double* pred_u, double* scratch, void* stream);

/* omg_closed_loop_step_der for a fleet of n_veh vehicles of one model and one spline basis in
 * each row of x (a multi-vehicle problem, reference Problem.simulate / predict looping over
 * self.vehicles, problem.py:187-192): vehicle v's n_input input splines are the columns of
 * length L at x[b, veh_off[v] + c*L].  HOST int32 veh_off [n_veh].  DEVICE plant_x, plant_u and
 * the four outputs are [B x n_veh x n_state | n_input]; scratch holds
 * B x n_veh x n_input x (n_traj + 24) doubles (disturb only).  One block of 32 threads per
 * (instance, vehicle).  The noise of vehicle v's input j is keyed by (seed, step, b, v*n_input + j,
 * sample pair): vehicle 0 draws what omg_closed_loop_step_der draws, and a realisation does not
 * depend on the batch size.  With n_veh = 1 and veh_off = {0} the outputs are
 * omg_closed_loop_step_der's, bit for bit (that entry point launches the same kernel).  Rejected
 * with a message: everything omg_closed_loop_step_der rejects, n_veh < 1, a null veh_off, and an
 * offset < 0 or with veh_off[v] + n_input*L > n. */
int omg_closed_loop_step_fleet(int32_t model, int32_t B, int32_t n_veh, int32_t n_state, int32_t n_input,
                               int32_t n, const double* x, const int32_t* veh_off, int32_t L,
                               int32_t n_samp, int32_t n_der, const double* R, double sample_time,
                               int32_t lag, double time_constant, int32_t disturb, int32_t n_traj,
                               const double* filt, const double* mean, const double* stdev,
                               uint64_t seed, int32_t step, const double* plant_x,
                               const double* plant_u, double* plant_x_next, double* plant_u_next,
                               double* pred_x, double* pred_u, double* scratch, void* stream);

/* omg_closed_loop_step_der with a free motion time (reference FreeTPoint2point.store / simulate,
 * point2point.py:313-346, on Vehicle.store / predict / simulate): every instance samples its own
 * plan on its own time axis, so no basis row is shared and the rows are built on the device.
 * DEVICE: x [B x n], plant_x, plant_u, the four outputs and scratch as omg_closed_loop_step_der;
 * scratch holds B x n_input x (max n_traj + 24) doubles (disturb only).  The input splines are
 * the first n_input columns of ONE spline block described as omg_eval_batch describes it:
 * spl_offset in x, basis length L, n_cols columns, degree, HOST knots [L + degree + 1].
 * Instance b reads its motion time T_b = x[b, t_index] on the device and takes its planned input
 * at samples s = 0..n_samp[b] from the values and derivatives of the columns at s*sample_time /
 * T_b, derivative d divided by T_b^d (the rows of the reference's store on
 * linspace(0, (n_traj-1)*sample_time, n_traj)), through the model's input map
 * (omg_closed_loop_step_der; n_der from the model's to 4, at most degree + 1).
 * HOST int32 n_samp [B]: samples of the update of b, min(update_time, T_b) / sample_time; 0 =
 * nothing is written for b (a stopped instance, or T_b below the sample time).  HOST int32
 * n_traj [B] (read with disturb only): length of b's stored trajectory, T_b / sample_time + 1,
 * over which its disturbance is filtered; 0 = no disturbance for b.  The noise is keyed by
 * (seed, step, b, signal, pair) with b the row of x: a realisation belongs to the instance and
 * does not depend on which other rows are stepped.  Filter, lag and RK4 are
 * omg_closed_loop_step_der's.  Rejected with a message: everything omg_closed_loop_step_der
 * rejects, a spline block outside x or with fewer than n_input columns, t_index outside x,
 * n_samp[b] < 0, 0 < n_traj[b] <= 12 (filtfilt's padding), 0 < n_traj[b] < n_samp[b] + 1, and
 * (max n_samp + 1) * n_input > 2048. */
int omg_closed_loop_step_free(int32_t model, int32_t B, int32_t n_state, int32_t n_input, int32_t n,
                              const double* x, int32_t spl_offset, int32_t L, int32_t n_cols,
                              int32_t degree, const double* knots, int32_t t_index, int32_t n_der,
                              const int32_t* n_samp, const int32_t* n_traj, double sample_time,
                              int32_t lag, double time_constant, int32_t disturb, const double* filt,
                              const double* mean, const double* stdev, uint64_t seed, int32_t step,
                              const double* plant_x, const double* plant_u, double* plant_x_next,
                              double* plant_u_next, double* pred_x, double* pred_u, double* scratch,
                              void* stream);

/* ADMM consensus step for n_agents agents on the current device (DEVICE pointers):
 * closed-form z-update, lambda-update and squared residuals of the reference's
 * ADMM updater (omgtools/problems/admm.py:117-168 construct_upd_z/update_z,
 * 248-266 upd_l, 268-307 upd_res; C++ twin ADMMPoint2Point::update2,
 * ADMMPoint2Point.cpp:213-265).  nsh shared coefficients per agent (n_spl
 * splines of L coefficients), n_nghb neighbours; PzT [nz x nz] is the TRANSPOSED
 * consensus projector (nz = nsh*(1+n_nghb)), c [n_agents x nz] its affine part,
 * Tf/Tb [L x L] the first-knot shift and its inverse.  z_*, l_* are updated in
 * place, res [n_agents x 3] receives (pr, dr, cr) squared.  The neighbour
 * exchange itself is the caller's NCCL step (problems/admm_gpu.py). */
int omg_admm_zl_update(int32_t n_agents, int32_t nsh, int32_t n_nghb, int32_t L,
                       const double* PzT, const double* c, const double* Tf,
                       const double* Tb, double rho,
                       const double* x_i, const double* x_j,
                       double* z_i, double* z_ij, double* l_i, double* l_ij,
                       double* res, void* stream);

/* ---- multi-GPU ADMM: the consensus exchange inside the boundary ----------------------------
 * The reference "communicates" by copying neighbours' fields in one process
 * (omgtools/problems/admm.py:468-475); its C++ export leaves the transport to the user
 * (update1 returns x_var and takes z_ji/l_ji, update2 takes x_j and returns z_ij/l_ij/
 * residuals: export/point2point/admm/ADMMPoint2Point.cpp:107-117, 213-265; the test shuffles
 * the vectors by hand, export/tests/formation/test.cpp:159-187).  Here one process per GPU
 * holds a contiguous slice of the agents and the transport is NCCL over NVLink:
 *
 *   omg_comm_unique_id   rank 0: 128 opaque bytes to hand to every rank (ncclGetUniqueId)
 *   omg_comm_create      every rank: join the communicator on `device` (ncclCommInitRank);
 *                        n_ranks = 1 needs no id and no NCCL
 *   omg_admm_exchange_x  after the x-update: x_j[i][k] <- x_i of agent nghb[i][k]
 *                        (ncclAllGather of the local x_i + an index kernel)
 *   omg_admm_zl_update_dist  omg_admm_zl_update, then ncclAllReduce of the three residual
 *                        sums and the second exchange z_ji[i][k] <- z_ij[nghb[i][k]][back[i][k]]
 *                        (likewise l) -- one stream-ordered call, no host synchronisation
 *
 * nghb / back are DEVICE int32 [n_local x n_nghb]: global agent id of neighbour k of local agent
 * i, and the position of agent i in that neighbour's own list.  Every rank holds n_local agents
 * (rank r: agents r*n_local ..).  NCCL is bound at run time (dlopen of libnccl.so.2, the copy a
 * host process such as PyTorch already loaded if any): the library has no link-time dependency
 * on it, and a single-GPU caller never touches it. */
typedef struct omg_comm omg_comm;
int omg_comm_unique_id(void* id128);
omg_comm* omg_comm_create(const void* id128, int32_t n_ranks, int32_t rank, int32_t device);
void omg_comm_destroy(omg_comm* c);
int omg_admm_exchange_x(omg_comm* c, int32_t n_local, int32_t nsh, int32_t n_nghb,
                        const int32_t* nghb, const double* x_i, double* x_j, void* stream);
int omg_admm_zl_update_dist(omg_comm* c, int32_t n_local, int32_t nsh, int32_t n_nghb, int32_t L,
                            const double* PzT, const double* cvec, const double* Tf,
                            const double* Tb, double rho, const double* x_i, const double* x_j,
                            double* z_i, double* z_ij, double* l_i, double* l_ij, double* res,
                            const int32_t* nghb, const int32_t* back, double* z_ji, double* l_ji,
                            double* res_total, void* stream);

/* Table files: the on-disk form of omg_tables, the stand-in for the nlp.c / nlp.so
 * bundle that the reference's exporter writes for its C++ runtime
 * (omgtools/export/export_p2p.py:43-60 -> Point2Point.cpp:80-91 nlpsol("problem",
 * "ipopt","nlp.so")).  A file is "OMGTBL\0\0", int32 abi_version, int32 record
 * count, then named records {char name[24]; int32 dtype (0 int32, 1 float64);
 * int32 pad; int64 count; data}.  Written by omg_tools_b200.solver.b200.save_tables;
 * omg_tables_read returns a heap object that owns its arrays (release it with
 * omg_tables_free) or NULL (omg_last_error).  Host only, no GPU needed. */
omg_tables* omg_tables_read(const char* path);
void omg_tables_free(omg_tables* tables);

/* ---- device-resident receding-horizon update ------------------------------------------------
 * The batched counterpart of the reference's exported Point2Point::update()
 * (omgtools/export/point2point/Point2Point.cpp:119-231) for a fixed-horizon Point2point with one
 * Holonomic or Holonomic3D vehicle (n_dim position splines; state = their values, input = their
 * derivatives / horizon) and obstacles that are static, move with x/v/a or rotate with theta.
 * One omg_mpc_update advances B independent instances, each on its own time t_b (B copies of
 * Point2Point), stream-ordered: after the first update of a handle it makes no synchronous CUDA
 * call and no allocation, so a sequence of updates can be captured in a CUDA graph.
 *
 * Per instance b, with round6(x) = rint(x * 1e6) / 1e6 (numpy.round(x, 6)), t_rel = round6(t_b)
 * mod knot_time, and a knot crossed when trunc(round6(t_prev_b / knot_time)) <
 * trunc(round6(t_b / knot_time)):
 *   prepare  cold start when |t_b| <= 1e-6 or the instance was flagged by omg_mpc_recover:
 *            state0 = the caller's state0[b], input0 = 0 (Holonomic::setInitialConditions), and
 *            the x row is x_template with the vehicle's columns set to linspace(state0, stateT, L)
 *            (getInitSplineValue).  Otherwise the prediction made when the last successful plan
 *            was committed: ideal: the plan's value and derivative / horizon at
 *            t_rel_prev + update_time; integrate: classical RK4 from the caller's state0[b]
 *            (the measured state at the start of that plan) over the plan's inputs at the
 *            update_time / sample_time + 1 samples from t_rel_prev, on the linearly interpolated
 *            input (the integration of omg_closed_loop_step's predict half, which is what the
 *            reference's Python predict does with odeint; Vehicle.cpp's predict takes the stage
 *            inputs instead), input0 = the planned input at the last sample.  At a knot crossing
 *            every shift block is multiplied by its T matrix (omg_shift_batch).  P[b] is
 *            p_template with state0, input0, poseT = stateT[b], t = t_rel, T = horizon and the
 *            obstacles' x, v, a (and theta) written in.
 *   solve    omg_solve_batch with the problem's own bounds, shared by all instances (with obstacles
 *            attached: each instance's own bound row, see omg_mpc_attach_obstacles).
 *   commit   status 0: the x row takes the solution, t_prev_b = t_b, state_traj[b] and
 *            input_traj[b] receive the plan's values and derivatives / horizon at
 *            t_rel + k * sample_time (k < trajectory_length; a sample past the horizon reads 0),
 *            the next prediction is stored and t_b = round6(t_b + update_time).  Any other
 *            status: t_prev_b = t_b (the next update does not shift again), the x row keeps the
 *            warm start it was solved from, t_b and the output rows are left as they were
 *            (Point2Point::update returns false).  status[b] and iters[b] are always written.
 * Obstacles are supplied on every call in their current state (the reference's obstacle_t):
 * obstacles[b] holds n_obs records of 3 * n_dim + 1 doubles, {x, v, a, theta}; theta is read only
 * for a rotating obstacle.  The rest of obstacle_t, each obstacle's shape (checkpoints and radii) and
 * its avoid flag (updateBounds), is per-instance state set by omg_mpc_set_obstacles after
 * omg_mpc_attach_obstacles (below).  A free motion time (FreeTPoint2point) has its own descriptor and
 * create call below and shares every other call.  Not covered: several vehicles, other vehicles,
 * time-based constraint shutdown, predict_shift and provide_prediction. */
typedef struct omg_mpc omg_mpc;   /* opaque handle */

typedef struct omg_mpc_desc {
  int32_t n, n_par;               /* the problem's sizes */
  int32_t n_dim;                  /* vehicle: states = inputs = position splines, 1 .. 3 */
  int32_t spl_offset;             /* column c of the vehicle's splines at x[spl_offset + c * L] */
  int32_t L, degree;              /* the vehicle's B-spline basis on [0, 1] */
  const double* knots;            /* [L + degree + 1] */
  double horizon, knot_time, update_time, sample_time;
  int32_t p_state0, p_input0, p_poseT, p_t, p_T;   /* offsets in p */
  int32_t n_obs;
  const int32_t* obs_kind;        /* [n_obs] 0: x, v, a; 1: x, v, a and theta (rotating) */
  const int32_t* obs_off;         /* [n_obs * 4] offsets in p of x, v, a, theta (-1: none) */
  int32_t n_shift;                /* warm-start shift blocks (father.shifted_entries()) */
  const int32_t* shift_off;       /* [n_shift] offset in x */
  const int32_t* shift_len;       /* [n_shift] basis length len */
  const int32_t* shift_ncol;      /* [n_shift] columns */
  const double* shift_T;          /* the n_shift row-major len x len matrices, concatenated */
  const double* x_template;       /* [n] father.get_variables().cat */
  const double* p_template;       /* [n_par] father.set_parameters(0.).cat */
} omg_mpc_desc;

enum { OMG_MPC_PREDICT_IDEAL = 0, OMG_MPC_PREDICT_INTEGRATE = 1 };

/* MPC files: "OMGMPC\0\0", int32 abi_version, int32 record count, then records in the format of
 * the table file, named after the fields of omg_mpc_desc (float64 scalars as records of one
 * double).  Written by omg_tools_b200.solver.b200.save_mpc.  omg_mpc_read returns a heap object
 * that owns its arrays (release it with omg_mpc_free_desc) or NULL (omg_last_error). */
omg_mpc_desc* omg_mpc_read(const char* path);
void omg_mpc_free_desc(omg_mpc_desc* desc);

/* Allocate the loop's state for B instances of `problem` on its device (the handle keeps a
 * pointer to the problem, which must outlive it).  prediction: OMG_MPC_PREDICT_*.  Returns NULL
 * with a message for: a null argument, n or n_par that differ from the problem's, B <= 0,
 * trajectory_length < 1 or above horizon / sample_time, an update_time that is not a positive
 * multiple of sample_time, an unknown prediction, and descriptor entries outside x or p. */
omg_mpc* omg_mpc_create(omg_problem* problem, const omg_mpc_desc* desc, int32_t B,
                        int32_t trajectory_length, int32_t prediction);
void omg_mpc_destroy(omg_mpc* mpc);

/* One update of every instance (see above).  DEVICE buffers: state0, stateT [B][n_dim],
 * obstacles [B][n_obs][3 n_dim + 1] (may be NULL when n_obs = 0), state_traj, input_traj
 * [B][trajectory_length][n_dim], status, iters [B].  Asynchronous on `stream`. */
int omg_mpc_update(omg_mpc* mpc, const double* state0, const double* stateT, const double* obstacles,
                   double* state_traj, double* input_traj, int32_t* status, int32_t* iters, void* stream);
/* Same call with HOST buffers (synchronous). */
int omg_mpc_update_host(omg_mpc* mpc, const double* state0, const double* stateT, const double* obstacles,
                        double* state_traj, double* input_traj, int32_t* status, int32_t* iters);
/* Cold-start the instances with mask[b] != 0 (HOST int32 [B]) on their next update, as
 * Point2Point::recover().  Synchronous: the flags are set when the call returns. */
int omg_mpc_recover(omg_mpc* mpc, const int32_t* mask);
/* ---- free motion time (FreeTPoint2point): T is a decision variable ----------------------------
 * The same handle type, created by omg_mpc_create_freet; omg_mpc_update(_host), omg_mpc_recover,
 * omg_mpc_time, omg_mpc_motion_time, omg_mpc_last_problem and omg_mpc_destroy serve both kinds.
 * Per instance b, with T_b the motion time of its last accepted plan (x[t_index]), dt =
 * update_time, st = sample_time and round6 as above:
 *   prepare  cold start on the first update and after omg_mpc_recover (a stopped instance
 *            included): x_template with linspace(state0, stateT, L) in the vehicle's columns
 *            and the template's T, state0 = the caller's state0[b], input0 = 0.
 *            After an accepted solve: the prediction from that plan on its own time axis
 *            (ideal: value and derivative / T_b at min(dt, T_b) / T_b; integrate: classical RK4
 *            from the caller's state0[b] over the planned inputs at s st / T_b, s = 0 ..
 *            round6(min(dt, T_b) / st), linearly interpolated, input0 = the last of them), then
 *            the stop test: the instance stops when T_b < dt, or when |state0 - stateT[b]| <=
 *            stop_tol and |input0| <= stop_tol (holonomic.py check_terminal_conditions).  A
 *            running instance is shifted from its plan's T (FreeTPoint2point.init_step):
 *            u, target = (dt, T_b - dt), or (T_b - dt, T_b) when T_b < 2 dt; tau = u / target;
 *            every block is re-expressed on shift_spline's basis (omg_shift_free_batch's
 *            arithmetic) when 0 < tau < 1, and x[t_index] = target.
 *            After a failed solve: no shift, the same warm start and stored prediction.
 *            P[b] is p_template with state0, input0, poseT = stateT[b] and the obstacles written
 *            in (t stays 0; there is no T parameter).
 *   solve    omg_solve_batch_rows on the instances that are not stopped.
 *   commit   a stopped instance: status OMG_MPC_STOPPED, 0 iterations; its time, warm start,
 *            motion time and output rows stay as they are until omg_mpc_recover.  Status 0: the
 *            x row takes the solution, state_traj[b] / input_traj[b] row j are the plan's value
 *            and derivative / T at min(j st, T) / T (rows past the plan hold its final point),
 *            the next prediction's samples are stored and t_b = round6(t_b + dt).  Any other
 *            status: as with a fixed horizon (the warm start, time and output rows are kept).
 * After the first update an update makes no synchronous call and no allocation, so updates stay
 * capturable in a CUDA graph, across the updates at which instances stop too. */
enum { OMG_MPC_STOPPED = -1 };    /* status of an instance not solved because it has stopped */

typedef struct omg_mpc_freeT_desc {
  int32_t n, n_par;               /* the problem's sizes */
  int32_t n_dim;                  /* vehicle: states = inputs = position splines, 1 .. 3 */
  int32_t spl_offset;             /* column c of the vehicle's splines at x[spl_offset + c * L] */
  int32_t L, degree;              /* the vehicle's B-spline basis on [0, 1] */
  const double* knots;            /* [L + degree + 1] */
  double update_time, sample_time;
  double stop_tol;                /* the vehicle's stop_tol */
  int32_t t_index;                /* offset of the motion time T in x */
  int32_t p_state0, p_input0, p_poseT;   /* offsets in p */
  int32_t n_obs;
  const int32_t* obs_kind;        /* [n_obs] as in omg_mpc_desc */
  const int32_t* obs_off;         /* [n_obs * 4] */
  int32_t n_blocks;               /* the spline blocks the warm start re-expresses */
  const int32_t* blk_off;         /* [n_blocks] offset in x */
  const int32_t* blk_len;         /* [n_blocks] basis length L */
  const int32_t* blk_ncol;        /* [n_blocks] columns */
  const int32_t* blk_degree;      /* [n_blocks] degree p */
  const double* blk_knots;        /* the n_blocks knot vectors [L + p + 1], concatenated */
  const double* x_template;       /* [n] father.get_variables().cat (holds the initial T) */
  const double* p_template;       /* [n_par] father.set_parameters(0.).cat */
} omg_mpc_freeT_desc;

/* MPC files of the free-T descriptor: the container of omg_mpc_read with records named after the
 * fields of omg_mpc_freeT_desc (written by omg_tools_b200.solver.b200.save_mpc_freeT).  Each
 * reader refuses the other kind's file, naming the other reader. */
omg_mpc_freeT_desc* omg_mpc_freet_read(const char* path);
void omg_mpc_freet_release(omg_mpc_freeT_desc* desc);

/* Returns NULL with a message for what omg_mpc_create rejects (but the horizon and knot time),
 * t_index outside x, a block outside x or beyond OMG_SPL_MAX_DEGREE / OMG_SPL_MAX_LEN, knots that
 * decrease, stop_tol < 0 and trajectory_length outside 1 .. (template T) / sample_time. */
omg_mpc* omg_mpc_create_freet(omg_problem* problem, const omg_mpc_freeT_desc* desc, int32_t B,
                              int32_t trajectory_length, int32_t prediction);

/* Each instance's T of its last accepted plan (the template's before the first) into DEVICE
 * T_out [B]; the horizon for a fixed-horizon handle.  Asynchronous on `stream`. */
int omg_mpc_motion_time(omg_mpc* mpc, double* T_out, void* stream);

/* Current time t_b of every instance into HOST t_out [B] (synchronises the device). */
int omg_mpc_time(omg_mpc* mpc, double* t_out);
/* The warm start and parameter rows handed to the last solve, DEVICE x0_out [B][n] and p_out
 * [B][n_par] (either may be NULL).  Asynchronous on `stream`. */
int omg_mpc_last_problem(omg_mpc* mpc, double* x0_out, double* p_out, void* stream);

/* ---- obstacle shapes and avoidance (the rest of the reference's obstacle_t) ------------------
 * Point2Point::update() takes, per obstacle, its checkpoints and radii, written into the parameters
 * on every call (export.py _create_fillParameterDict), and an avoid flag: when it is false,
 * updateBounds sets the bounds of that obstacle's own constraint rows to -inf / +inf for the solve
 * (export.py _create_updateBounds; Point2Point.cpp:213-218).  The hyperplane rows of the
 * environment and the vehicle's own rows are not among them.  Here both are per-instance state of a
 * handle of either kind: once attached, every update writes instance b's stored shapes into P[b]
 * after the template (and the obstacles' x, v, a, theta) and solves with instance b's own bound row.
 *
 * The descriptor lists the obstacles in environment order (the order of omg_mpc_desc's obs_off). */
typedef struct omg_mpc_obstacles_desc {
  int32_t n_obs;
  const int32_t* chk_off;         /* [n_obs] offset in p of the checkpoints x0, y0, x1, y1, ... */
  const int32_t* chk_len;         /* [n_obs] n_chk * n_dim */
  const int32_t* rad_off;         /* [n_obs] offset in p of the radii */
  const int32_t* rad_len;         /* [n_obs] n_chk */
  const int32_t* row_off;         /* [n_obs] first g row of the obstacle's own constraints */
  const int32_t* row_len;         /* [n_obs] their number */
} omg_mpc_obstacles_desc;

/* Obstacle files: the container of omg_mpc_read under the magic "OMGOBS\0\0", records named after
 * the fields of omg_mpc_obstacles_desc (written by omg_tools_b200.solver.b200.save_mpc_obstacles).
 * Returns a heap object (release it with omg_mpc_obstacles_release) or NULL (omg_last_error). */
omg_mpc_obstacles_desc* omg_mpc_obstacles_read(const char* path);
void omg_mpc_obstacles_release(omg_mpc_obstacles_desc* desc);

/* Allocate and initialise the handle's per-instance obstacle state: every shape is the template's
 * (p_template at chk_off / rad_off), every avoid flag is set, and each instance's bound row [m] is
 * the tables' bounds.  Synchronous; call it once, before updates that are captured in a graph.
 * Returns -1 with a message for: a null argument, an n_obs that differs from the handle's, p entries
 * outside p, a checkpoint length other than n_dim times the radius length (which must be >= 1),
 * row ranges outside [0, m) or overlapping, a row in a range whose table bounds are an equality
 * (the equality rows are part of the solver's symbolic analysis), and a handle that already has
 * obstacles attached. */
int omg_mpc_attach_obstacles(omg_mpc* mpc, const omg_mpc_obstacles_desc* desc);

/* Set the obstacles' shapes and avoid flags of every instance until the next set call (updates and
 * omg_mpc_recover leave them as they are).  DEVICE buffers: shapes [B][sum_k (n_dim + 1) n_chk_k],
 * per obstacle its checkpoints (chk_len doubles) and then its radii (rad_len), the field order of
 * obstacle_t; avoid [B][n_obs], nonzero: avoid.  Either may be NULL, which keeps that part.
 * Asynchronous on `stream` and capturable in a CUDA graph.  Returns -1 when no obstacles are
 * attached. */
int omg_mpc_set_obstacles(omg_mpc* mpc, const double* shapes, const int32_t* avoid, void* stream);
/* Same call with HOST buffers (synchronous). */
int omg_mpc_set_obstacles_host(omg_mpc* mpc, const double* shapes, const int32_t* avoid);

const char* omg_last_error(void);
int omg_abi_version(void);

#ifdef __cplusplus
}
#endif
#endif /* OMG_B200_H */
