// omg_b200.cu -- batched primal-dual interior-point solve of OMG-tools' spline
// NLP on H100 (sm_90a).  One thread block per problem instance (persistent
// blocks pull instances from a counter; 2 x 256 threads or 1 x 512 per SM); the
// per-instance state (KKT envelope, Jacobian values, iterate vectors) lives in
// shared memory for the duration of the solve, constant tables stream from L2.
// Kernel variants: omg_ipm_kernel / _2cta (everything in shared memory) and
// omg_ipm_kernel_xl / _xl_2cta (problems with shared intermediates or structures
// larger than one SM's shared memory: tape, chain-rule slots and, if needed, the
// KKT envelope in an L2-resident per-block scratch).
//
// Replaces the CasADi+IPOPT call of the reference (omgtools/problems/
// problem.py:113, optilayer.py:49-60).  Algorithm = oracle/ipm_ref.py (IPOPT
// semantics, Waechter & Biegler 2006); tables = basics/lowering.py.
//
// Design rules (a dependent global load costs many times a shared-memory load, a
// shuffle or a block barrier; tools/ubench/lat.cu measures them on the GPU at hand):
//   * no dependent chains through global memory: every pass reads one record
//     per work item (row / column / H position / W slot) and then streams
//     contiguous 32-byte term records with independent loads;
//   * the sequential part of the factorisation (8x8 diagonal blocks, 8x8
//     triangular solves) runs in the registers of a single thread -- no
//     shuffles, little code;
//   * shared-memory placement is adaptive: arrays that do not fit fall back to
//     an L2-resident per-block scratch (generic pointers, same code path).
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <math.h>
#include <algorithm>
#include <string>
#include <vector>

#include "../../include/omg_b200.h"

// The same source also builds with g++ as a functional CPU emulation of the kernels
// (tools/cpu_emu: its cuda_runtime.h stand-in defines OMG_CPU_EMU and these two macros;
// test infrastructure for a GPU-less container, never loaded by the product).
#ifndef OMG_CPU_EMU
#define OMG_DYN_SHARED(name) extern __shared__ __align__(16) double name[]
#define OMG_LAUNCH(kern, grid, block, smem, stream, ...) kern<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__)
#else
#define __grid_constant__
#endif

#define NT ((int)blockDim.x)   // threads per block: 512 (1 block/SM) or 256 (2 blocks/SM)
#define NWARP (NT / 32)
#define MAX_NT 512
#define MAX_NWARP (MAX_NT / 32)
#define NB 8              // panel width (== lowering.KKT_NB)
#define MAXF 32           // filter capacity
#define NRED 12           // values per fused block reduction
#define NRED_OPS OP_MAX, OP_MAX, OP_MIN, OP_MAX, OP_MAX, OP_MAX, OP_SUM, OP_SUM, OP_SUM, OP_SUM, OP_MAX, OP_SUM
#define FULL 0xffffffffu
#define TRACE_COLS 8
#define TRACE_ROWS 512
#define MAXW 5            // max x-factors per term record

// ---------------------------------------------------------------------------
// table records (device)
// ---------------------------------------------------------------------------
struct __align__(16) PTerm {       // 32 bytes: coef * V[cidx] * prod x_ext[x[k]]
  double coef;
  unsigned short cidx, aux;        // aux: lambda row (W terms) or slot offset in row (J terms)
  unsigned short x[MAXW];
  unsigned short pad[5];
};
struct __align__(16) RowRec { int g0, g1, jt0, jt1, s0, ns, pad0, pad1; };  // per constraint row
struct __align__(16) HqRec { int dst, p0, p1, diag; };                      // per H position
struct __align__(16) WRec { int dst, t0, t1, pad; };                        // per Hessian slot

enum { A_JVAL = 0, A_SIG, A_JSV, A_G, A_S, A_Y, A_ZU, A_DSC, A_SU, A_DS, A_DY, A_DZU, A_GT,
       A_ST, A_WV, A_ZL, A_SL, A_DZL, A_BEQ, N_ARR };

struct DevTab {
  int n, m, n_par, n_v, n_tape, n_levels, nnz_j, nnz_w, nnz_h, n_eq, N;
  int env_size, n_panels, max_panel_rows, n_panel_rows, n_f;
  const int *tape_func, *tape_ptr, *tape_fac, *level_ptr; const double* tape_coef;
  const PTerm *Gt, *Jt, *Wt, *Ft, *DFt;
  const RowRec* rowrec; const WRec* wrec; const HqRec* hq; const unsigned* hpack;
  const int *dfptr;                     // [n+1] grad-f term ranges per column
  const int *colptr; const unsigned* colrec;   // CSC of J: slot | row << 16
  const unsigned short* jcol16;         // [nnz_j] column of each slot
  const int *eq_rows, *pos_var, *pos_eq, *ksign, *env_first, *env_ptr, *jdst, *kdiag,
            *panel_ptr, *panel_rows, *panel_cmin;
  // intermediates (XL kernel only): G term ranges of the mids, term ranges of the extra
  // J slots (A = d row/d mid, C = d mid/d x), chain-rule pair lists, mu = A^T lambda lists
  int n_mid, nnz_jx, n_hq_heavy;
  const int2* midg; const int* jtptr; const int* jrow;
  const int *jp_ptr, *jp_a, *jp_c, *mu_ptr, *mu_row, *mu_slot;
  const int* jxvar; int n_jxvar;       // extra J slots with an x factor (the others are constant in a solve)
  // extra Hessian slots (mid coefficient depends on x or on another mid): wrec[nnz_w ..
  // nnz_w+nnz_wx) hold the term ranges, xq the H positions that gather
  // sum Wx[e.x] * Jx[e.y] * (e.z >= 0 ? Jx[e.z] : 1)
  int nnz_wx, n_xq;
  const HqRec* xq; const int4* xqp;
};

struct Smem {                      // offsets in doubles
  int K, Pt, PtS, Ld, xe, xt, dx, u, gf, diag0, invd, V, red, filt, rbase, rt8;
  int sgn, eptr, efirst, pptr, prow, pcmin;
  int arr[N_ARR];                  // >= 0: shared offset; < 0: -(scratch offset + 1)
  int LDP, total;
  int Kg, Vg, jxg, mug, Kcg, wxg;  // XL kernel: scratch offsets (K only if S.K < 0)
};

struct Batch {
  int B; int bounds_shared;
  const double *x0, *p, *lbg, *ubg, *lam0;
  double *x, *lam, *f; int *status, *iters;
  double* dscr; int* iscr; int dscr_stride, iscr_stride;
  int* counter; double* trace;
  // optional row list: instance i of the counter is row rows[i], for i < *n_rows (both null: row i
  // for i < B).  Rows index x0, p, the bounds and every output.
  const int* rows; const int* n_rows;
};

// The row the persistent grid takes next (thread 0 of a block); B when none is left.
__device__ __forceinline__ int omg_next_row(const Batch& A) {
  const int i = atomicAdd(A.counter, 1);
  if (!A.rows) return i;
  return i < *A.n_rows ? A.rows[i] : A.B;
}

struct Ctl {                       // uniform per-block control scalars
  double mu, tau, theta_max, theta_min, delta_w, delta_w_last, delta_c;
  double alpha, theta, phi, f, fsc;
  int n_eq, n_bounds, iter, status, fail, eq_fail, first_try, nfilt, inst, n_restart;
};

// IPOPT constants not exposed as options (oracle/ipm_ref.py DEFAULTS)
#define KAPPA_EPS 10.0
#define KAPPA_MU 0.2
#define THETA_MU 1.5
#define TAU_MIN 0.99
#define S_MAX 100.0
#define KAPPA_SIGMA 1e10
#define GAMMA_THETA 1e-5
#define GAMMA_PHI 1e-8
#define ETA_PHI 1e-8
#define S_THETA 1.1
#define S_PHI 2.3
#define DELTA_LS 1.0
#define GAMMA_ALPHA 0.05
#define THETA_MAX_FACT 1e4
#define THETA_MIN_FACT 1e-4
#define DELTA_W0 1e-4
#define DELTA_W_MIN 1e-20
#define DELTA_W_MAX 1e40
#define KAPPA_W_PLUS_FIRST 100.0
#define KAPPA_W_PLUS 8.0
#define KAPPA_W_MINUS (1.0 / 3.0)
#define DELTA_C_VAL 1e-8
#define DELTA_C_EXP 0.25
#define PIV_TOL 1e-12
#define INF_BOUND 1e19
#define MAX_LS 40
#define SOFT_RESTO_FACTOR 0.9999
#define DBL_EPS 2.220446049250313e-16

enum { OP_MAX = 0, OP_MIN = 1, OP_SUM = 2 };

// phase timers (debug, opt.trace=1, instance 0): cycles per phase summed over the solve
#define NPHASE 16
#define TICK(k) do { if (tracing && threadIdx.x == 0) { const long long t_ = clock64(); \
  phase_cyc[k] += (double)(t_ - phase_t0); phase_t0 = t_; } } while (0)

__device__ __forceinline__ double term_value(const PTerm* __restrict__ p, const double* __restrict__ V,
                                             const double* __restrict__ xe, int* aux) {
  const uint4 a = __ldg(reinterpret_cast<const uint4*>(p));
  const uint4 b = __ldg(reinterpret_cast<const uint4*>(p) + 1);
  double v = __hiloint2double((int)a.y, (int)a.x) * V[a.z & 0xffffu];
  *aux = (int)(a.z >> 16);
  v *= xe[a.w & 0xffffu]; v *= xe[a.w >> 16];
  v *= xe[b.x & 0xffffu]; v *= xe[b.x >> 16];
  v *= xe[b.y & 0xffffu];
  return v;
}

__device__ __forceinline__ double eval_range(const PTerm* __restrict__ t, int lo, int hi,
                                             const double* __restrict__ V, const double* __restrict__ xe) {
  double acc = 0.0;
  int aux;
#pragma unroll 4
  for (int k = lo; k < hi; ++k) acc += term_value(t + k, V, xe, &aux);
  return acc;
}

template <int OP>
__device__ __forceinline__ double red_op(double a, double b) {
  return (OP == OP_MAX) ? fmax(a, b) : (OP == OP_MIN) ? fmin(a, b) : a + b;
}

// Fused block reduction of the values v[r], slot r combined by OPS[r] (a compile-time choice,
// so each slot costs one instruction per step and no branches); every thread returns with the
// results.  Order per slot: lane shuffles, then warps 0..NWARP-1.
template <int... OPS>
__device__ __forceinline__ void block_reduce(double (&v)[sizeof...(OPS)], double* red) {
  constexpr int NR = sizeof...(OPS);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    int r = 0;
    ((v[r] = red_op<OPS>(v[r], __shfl_down_sync(FULL, v[r], off)), ++r), ...);
  }
  if (lane == 0) {
#pragma unroll
    for (int r = 0; r < NR; ++r) red[warp * NR + r] = v[r];
  }
  __syncthreads();
#pragma unroll
  for (int r = 0; r < NR; ++r) v[r] = red[r];
#pragma unroll 1
  for (int w = 1; w < NWARP; ++w) {
    int r = 0;
    ((v[r] = red_op<OPS>(v[r], red[w * NR + r]), ++r), ...);
  }
  __syncthreads();
}

__device__ __forceinline__ bool cmp_le(double lhs, double rhs, double base) {
  return lhs - rhs <= 10.0 * DBL_EPS * fabs(base);
}

OMG_DYN_SHARED(sm);

// shared-memory copies of the KKT structure arrays, addressed from the block's
// dynamic shared array so the compiler emits LDS (not generic loads)
#define KS_SGN    (sm + S.sgn)        // pivot signs S of K = L S L^T (rewritten by every factorisation)
#define KS_EPTR   (reinterpret_cast<const int*>(sm + S.eptr))
#define KS_EFIRST (reinterpret_cast<const int*>(sm + S.efirst))
#define KS_PPTR   (reinterpret_cast<const int*>(sm + S.pptr))
#define KS_PROW   (reinterpret_cast<const int*>(sm + S.prow))
#define KS_PCMIN  (reinterpret_cast<const int*>(sm + S.pcmin))

// ---------------------------------------------------------------------------
// Blocked right-looking factorisation K = L S L^T on envelope storage.
//   row i (permuted order) is stored from column first[i] (multiple of NB) to i
//   at K[env_ptr[i] + j - first[i]]; row N is the right-hand side (never a
//   pivot), so after the sweep it holds S L^{-1} r.
// Per 8-column panel: (1) ONE thread factors the 8x8 diagonal block in
// registers, (2) one thread per reached row does the panel solve, (3) the
// rank-8 trailing update runs over 2x2 register tiles of the reached rows.
// Pivot j must satisfy sign[j]*pivot > PIV_TOL*|K_jj| (variables) or > 0
// (equality rows); otherwise ctl->fail (eq_fail for an equality pivot).
// ---------------------------------------------------------------------------
// WIDE: a panel may reach more rows than the block has threads (max_panel_rows + 2 > NT); the
// rows from NT on then go to a loop strided by NT.  A separate instantiation, so the kernels of
// every other problem keep the code (and registers) of one row per thread.
template <bool WIDE>
__device__ __forceinline__ void factor_env(const DevTab& T, const Smem& S, double* K, Ctl* ctl, double* pc,
                                           const int mode) {
  const int tid = threadIdx.x;
  const int N = T.N;
  const int LDP = S.LDP;
  double* Pt = sm + S.Pt; double* PtS = sm + S.PtS; double* Ld = sm + S.Ld;
  const double* diag0 = sm + S.diag0; double* invd = sm + S.invd;
  int* rbase = reinterpret_cast<int*>(sm + S.rbase);
  int* rrow = rbase + LDP;
  double* sgn = KS_SGN; const int* eptr = KS_EPTR; const int* efirst = KS_EFIRST;
  int n_neg = 0;               // negative pivots so far (thread 0)
  const int* pptr = KS_PPTR; const int* prow = KS_PROW;
  long long t0 = clock64();
#define FT(k) do { if (pc && tid == 0) { const long long t_ = clock64(); pc[k] += (double)(t_ - t0); t0 = t_; } } while (0)
  for (int pb = 0; pb < T.n_panels; ++pb) {
    const int kb = pb * NB;
    const int nb = min(NB, N - kb);
    // ---- 1. diagonal block: staged into Ld (64 threads), factored by ONE thread in
    //         registers (branch-free pivots), scattered back by 64 threads ----------
    if (tid < NB * NB) {
      const int r = tid >> 3, c = tid & 7;
      double v = 0.0;
      if (r < nb && c <= r) v = K[eptr[kb + r] + kb - efirst[kb + r] + c];
      Ld[tid] = v;
    }
    __syncthreads();
    if (tid == 0) {
      double a[NB][NB];
#pragma unroll
      for (int r = 0; r < NB; ++r)
#pragma unroll
        for (int c = 0; c <= r; ++c) a[r][c] = Ld[r * NB + c];
      int bad_at = -1;
#pragma unroll
      for (int j = 0; j < NB; ++j) {
        // rows >= nb are zero-padded: give them a unit pivot so the arithmetic stays finite
        const bool live = (j < nb);
        // mode 0 (IPOPT's inertia test): S takes the sign of the pivot as it comes, only the
        // number of negative pivots is checked at the end; mode 1: S fixed (+ variables,
        // - equality rows), a pivot of the other sign fails
        // (|pivot| keeps the sign selection off the dependent chain pivot -> rsqrt -> column)
        const double sj = !live ? 1.0 : (mode ? sgn[kb + j] : (a[j][j] > 0.0 ? 1.0 : -1.0));
        const double d = !live ? 1.0 : (mode ? sj * a[j][j] : fabs(a[j][j]));
        const double thr = (live && (mode == 0 || sj > 0.0)) ? PIV_TOL * fmax(diag0[kb + j], 1e-300) : 0.0;
        const bool fail_j = !(d > thr) || !(d < 1e300);
        if (fail_j && bad_at < 0) bad_at = kb + j;
        if (live) { sgn[kb + j] = sj; n_neg += (sj < 0.0) ? 1 : 0; }
        const double inv = rsqrt(d);
        a[j][j] = d * inv;
        if (live) invd[kb + j] = inv;
        const double f = inv * sj;
#pragma unroll
        for (int r = j + 1; r < NB; ++r) a[r][j] *= f;
#pragma unroll
        for (int r = j + 1; r < NB; ++r) {
          const double lr = sj * a[r][j];
#pragma unroll
          for (int c = j + 1; c <= r; ++c) a[r][c] -= lr * a[c][j];
        }
      }
      if (bad_at >= 0) { ctl->fail = 1; ctl->eq_fail = (T.ksign[bad_at] < 0) ? 1 : 0; }
      else if (mode == 0 && n_neg > T.n_eq) { ctl->fail = 1; ctl->eq_fail = 0; }   // too many already: stop early
#pragma unroll
      for (int r = 0; r < NB; ++r)
#pragma unroll
        for (int c = 0; c <= r; ++c) Ld[r * NB + c] = a[r][c];
    }
    __syncthreads();
    if (!ctl->fail && tid < NB * NB) {
      const int r = tid >> 3, c = tid & 7;
      if (r < nb && c <= r) K[eptr[kb + r] + kb - efirst[kb + r] + c] = Ld[tid];
    }
    __syncthreads();
    FT(7);
    if (ctl->fail) return;
    // ---- 2. panel solve over the rows this panel reaches ----------------------
    const int p0 = pptr[pb];
    const int nrows = pptr[pb + 1] - p0;
    double2* P2 = reinterpret_cast<double2*>(Pt);
    double2* PS2 = reinterpret_cast<double2*>(PtS);
    auto solve_row = [&](const int rr) {
      const int r = prow[p0 + rr];
      const int rb = eptr[r] - efirst[r];
      rbase[rr] = rb; rrow[rr] = r;
      double* Kr = K + rb + kb;
      double a[NB], sg[NB];
#pragma unroll
      for (int c = 0; c < NB; ++c) { a[c] = (c < nb) ? Kr[c] : 0.0; sg[c] = (c < nb) ? sgn[kb + c] : 1.0; }
#pragma unroll
      for (int c = 0; c < NB; ++c) {
        if (c < nb) {
          double v = a[c];
#pragma unroll
          for (int j = 0; j < c; ++j) v -= sg[j] * a[j] * Ld[c * NB + j];
          a[c] = v * invd[kb + c] * sg[c];
        }
      }
#pragma unroll
      for (int c = 0; c < NB; ++c) if (c < nb) Kr[c] = a[c];
      // panel buffers as double2 [column pair][row]: conflict-free stores here, and
      // at most 2-way conflicts for the 2x2-tile loads of the trailing update
#pragma unroll
      for (int q = 0; q < NB / 2; ++q) {
        const double v0 = (2 * q < nb) ? a[2 * q] : 0.0, v1 = (2 * q + 1 < nb) ? a[2 * q + 1] : 0.0;
        P2[q * LDP + rr] = make_double2(v0, v1);
        PS2[q * LDP + rr] = make_double2(sg[2 * q] * v0, sg[2 * q + 1] * v1);
      }
    };
    auto zero_row = [&](const int rr) {   // zero padding rows nrows, nrows + 1 for the 2x2 tiles
#pragma unroll
      for (int q = 0; q < NB / 2; ++q) { P2[q * LDP + rr] = make_double2(0.0, 0.0); PS2[q * LDP + rr] = make_double2(0.0, 0.0); }
    };
    if (tid < nrows) solve_row(tid);
    else if (tid < nrows + 2 && tid < LDP) zero_row(tid);
    if constexpr (WIDE) {   // row rr on thread rr % NT
      for (int rr = tid + NT; rr < nrows + 2 && rr < LDP; rr += NT) {
        if (rr < nrows) solve_row(rr);
        else zero_row(rr);
      }
    }
    __syncthreads();
    FT(8);
    // ---- 3. trailing update: 2x2 tiles over list positions (a >= b) -----------
    const int nt2 = (nrows + 1) >> 1;
    const int W = nt2 + 1, H2 = (nt2 + 1) >> 1;
    for (int t = tid; t < H2 * W; t += NT) {
      const int ra = t / W, cb = t - ra * W;
      int ta, tb;
      if (cb <= ra) { ta = ra; tb = cb; }
      else { ta = nt2 - 1 - ra; tb = cb - ra - 1; if (ta == ra) continue; }
      const int a0 = ta * 2, b0 = tb * 2;
      const double2* A0 = reinterpret_cast<const double2*>(Pt) + a0;
      const double2* B0 = reinterpret_cast<const double2*>(PtS) + b0;
      double acc00 = 0.0, acc01 = 0.0, acc10 = 0.0, acc11 = 0.0;
#pragma unroll
      for (int q = 0; q < NB / 2; ++q) {
        const double2 x0 = A0[q * LDP], x1 = A0[q * LDP + 1], y0 = B0[q * LDP], y1 = B0[q * LDP + 1];
        acc00 += x0.x * y0.x; acc00 += x0.y * y0.y;
        acc01 += x0.x * y1.x; acc01 += x0.y * y1.y;
        acc10 += x1.x * y0.x; acc10 += x1.y * y0.y;
        acc11 += x1.x * y1.x; acc11 += x1.y * y1.y;
      }
      // scatter into K (only b <= a, column < N)
      const int la0 = a0, la1 = a0 + 1, lb0 = b0, lb1 = b0 + 1;
      const int c0 = rrow[lb0];
      const int c1 = (lb1 < nrows) ? rrow[lb1] : N;
      if (la0 < nrows) {
        const int rb = rbase[la0];
        if (lb0 <= la0 && c0 < N) K[rb + c0] -= acc00;
        if (lb1 <= la0 && c1 < N) K[rb + c1] -= acc01;
      }
      if (la1 < nrows) {
        const int rb = rbase[la1];
        if (lb0 <= la1 && c0 < N) K[rb + c0] -= acc10;
        if (lb1 <= la1 && c1 < N) K[rb + c1] -= acc11;
      }
    }
    __syncthreads();
    FT(9);
  }
#undef FT
  if (mode == 0 && tid == 0 && !ctl->fail && n_neg != T.n_eq) {   // Sylvester: wrong inertia
    ctl->fail = 1; ctl->eq_fail = (n_neg < T.n_eq) ? 1 : 0;
  }
}

// Back substitution L^T u = w on envelope storage (w = row N of L on entry).
__device__ __forceinline__ void back_solve_env(const DevTab& T, const Smem& S, const double* K) {
  const int tid = threadIdx.x;
  const int N = T.N;
  const double* invd = sm + S.invd; double* w = sm + S.u;
  const int* eptr = KS_EPTR; const int* efirst = KS_EFIRST; const int* pcmin = KS_PCMIN;
  for (int pb = T.n_panels - 1; pb >= 0; --pb) {
    const int kb = pb * NB;
    const int nb = min(NB, N - kb);
    // per-row bases of the block (uniform; 16 independent shared loads)
    int rbs[NB], rfs[NB];
#pragma unroll
    for (int j = 0; j < NB; ++j) {
      const int rj = min(kb + j, N - 1);
      rfs[j] = efirst[rj]; rbs[j] = eptr[rj] - rfs[j];
    }
    if (tid == 0) {        // 8x8 upper-triangular solve in registers
      double wv[NB], dinv[NB], L[NB][NB];
#pragma unroll
      for (int j = 0; j < NB; ++j) {
        wv[j] = (j < nb) ? w[kb + j] : 0.0;
        dinv[j] = (j < nb) ? invd[kb + j] : 1.0;
#pragma unroll
        for (int c = 0; c < j; ++c) L[j][c] = (j < nb) ? K[rbs[j] + kb + c] : 0.0;
      }
#pragma unroll
      for (int j = NB - 1; j >= 0; --j) {
        const double uj = wv[j] * dinv[j];
        wv[j] = uj;
#pragma unroll
        for (int c = 0; c < j; ++c) wv[c] -= L[j][c] * uj;
      }
#pragma unroll
      for (int j = 0; j < NB; ++j) if (j < nb) w[kb + j] = wv[j];
    }
    __syncthreads();
    const int cmin = pcmin[pb];
    for (int c = cmin + tid; c < kb; c += NT) {
      double l[NB], uu[NB];
#pragma unroll
      for (int j = 0; j < NB; ++j) {
        const bool in = (j < nb) && (c >= rfs[j]);
        l[j] = in ? K[rbs[j] + c] : 0.0;
        uu[j] = (j < nb) ? w[kb + j] : 0.0;
      }
      double acc0 = w[c], acc1 = 0.0;
#pragma unroll
      for (int j = 0; j < NB; j += 2) { acc0 -= l[j] * uu[j]; acc1 -= l[j + 1] * uu[j + 1]; }
      w[c] = acc0 + acc1;
    }
    __syncthreads();
  }
}

// Constraint Jacobian of the XL kernel, one thread per slot (rows differ widely in size).
// First the extra slots jx[s], s in [nnz_j, nnz_jx): A = d row/d mid (parameter-only) and
// C = d mid/d x; then every constraint slot = direct terms + chain rule
// sum_e A[jp_a[e]] * C[jp_c[e]], scaled by the row scaling dsc (nullptr: unscaled).
// Ends with a block barrier.
__device__ __forceinline__ void jac_xl(const DevTab& T, const double* __restrict__ V,
                                       const double* __restrict__ xe, double* jx, double* jval,
                                       const double* dsc, const bool first) {
  const int tid = threadIdx.x;
  if (first) {   // every extra slot; the parameter-only ones (A of config 4) keep this value
    for (int s = T.nnz_j + tid; s < T.nnz_jx; s += NT)
      jx[s] = eval_range(T.Jt, T.jtptr[s], T.jtptr[s + 1], V, xe);
  } else {
    for (int q = tid; q < T.n_jxvar; q += NT) {
      const int s = T.jxvar[q];
      jx[s] = eval_range(T.Jt, T.jtptr[s], T.jtptr[s + 1], V, xe);
    }
  }
  __syncthreads();
  for (int s = tid; s < T.nnz_j; s += NT) {
    double acc = eval_range(T.Jt, T.jtptr[s], T.jtptr[s + 1], V, xe);
    if (T.n_mid)
      for (int e = T.jp_ptr[s]; e < T.jp_ptr[s + 1]; ++e) acc += jx[T.jp_a[e]] * jx[T.jp_c[e]];
    jval[s] = dsc ? dsc[T.jrow[s]] * acc : acc;
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------
// the solver kernel
// ---------------------------------------------------------------------------
// XL = true: problems with intermediates (n_mid > 0) and/or a KKT envelope / parameter tape
// that exceeds shared memory: V (and K if needed) live in the block's L2-resident scratch.
template <bool XL, bool WIDE>
__device__ __forceinline__ void ipm_body(const DevTab& T, const omg_options& O, const Batch& A, const Smem& S) {
  __shared__ Ctl ctl;
  __shared__ double phase_cyc[NPHASE];
  double* const Dx = A.dscr + (size_t)blockIdx.x * A.dscr_stride;
  double* K = (XL && S.K < 0) ? Dx + S.Kg : sm + S.K;
  double* u = sm + S.u;
  double* xe = sm + S.xe;
  double* xt = sm + S.xt;
  double* dx = sm + S.dx;
  double* gf = sm + S.gf;
  double* diag0 = sm + S.diag0;
  double* V = (XL && S.V < 0) ? Dx + S.Vg : sm + S.V;
  double* jx = XL ? Dx + S.jxg - T.nnz_j : nullptr;   // indexed by slot id >= nnz_j
  double* mu_mid = XL ? Dx + S.mug : nullptr;
  double* wx = XL ? Dx + S.wxg : nullptr;        // values of the cross-Hessian slots
  double* Kc = Dx + S.Kcg;
  const int n_xe = T.n + 1 + (XL ? T.n_mid : 0);
  double* red = sm + S.red;
  double* filt = sm + S.filt;
  unsigned char* rt = reinterpret_cast<unsigned char*>(sm + S.rt8);
  const int tid = threadIdx.x;
  const int n = T.n, m = T.m;
  {  // KKT structure arrays -> shared memory (once per block)
    double* sgn = sm + S.sgn;
    int* eptr = reinterpret_cast<int*>(sm + S.eptr);
    int* efirst = reinterpret_cast<int*>(sm + S.efirst);
    int* pptr = reinterpret_cast<int*>(sm + S.pptr);
    int* prow = reinterpret_cast<int*>(sm + S.prow);
    int* pcmin = reinterpret_cast<int*>(sm + S.pcmin);
    for (int i = tid; i < T.N; i += NT) sgn[i] = (double)T.ksign[i];
    for (int i = tid; i < T.N + 2; i += NT) eptr[i] = T.env_ptr[i];
    for (int i = tid; i < T.N + 1; i += NT) efirst[i] = T.env_first[i];
    for (int i = tid; i < T.n_panels + 1; i += NT) pptr[i] = T.panel_ptr[i];
    for (int i = tid; i < T.n_panel_rows; i += NT) prow[i] = T.panel_rows[i];
    for (int i = tid; i < T.n_panels; i += NT) pcmin[i] = T.panel_cmin[i];
  }
  __syncthreads();

  // per-instance arrays: shared memory if they fit, else L2-resident scratch
  double* D = A.dscr + (size_t)blockIdx.x * A.dscr_stride;
#define ARR(k) ((S.arr[k] >= 0) ? (sm + S.arr[k]) : (D + (-(S.arr[k]) - 1)))
  double* jval = ARR(A_JVAL); double* sig = ARR(A_SIG); double* jsv = ARR(A_JSV);
  double* g = ARR(A_G); double* s = ARR(A_S); double* y = ARR(A_Y); double* zU = ARR(A_ZU);
  double* dsc = ARR(A_DSC); double* sU = ARR(A_SU); double* ds = ARR(A_DS); double* dy = ARR(A_DY);
  double* dzU = ARR(A_DZU); double* gt = ARR(A_GT); double* st = ARR(A_ST); double* wv = ARR(A_WV);
  double* zL = ARR(A_ZL); double* sL = ARR(A_SL); double* dzL = ARR(A_DZL); double* beq = ARR(A_BEQ);
#undef ARR
  int* I = A.iscr + (size_t)blockIdx.x * A.iscr_stride;
  int* eqidx = I;           int* eqrow = eqidx + m;

  for (;;) {
    // ---- fetch next instance ------------------------------------------------
    if (tid == 0) ctl.inst = omg_next_row(A);
    __syncthreads();
    const int inst = ctl.inst;
    if (inst >= A.B) return;
    const double* x0 = A.x0 + (size_t)inst * n;
    const double* par = A.p + (size_t)inst * T.n_par;
    const double* lbg = A.lbg + (A.bounds_shared ? 0 : (size_t)inst * m);
    const double* ubg = A.ubg + (A.bounds_shared ? 0 : (size_t)inst * m);
    const bool tracing = (O.trace != 0) && inst == 0 && A.trace != nullptr;
    long long phase_t0 = clock64();
    if (tracing && tid == 0) for (int k = 0; k < NPHASE; ++k) phase_cyc[k] = 0.0;

    // ---- S1: parameter tape ---------------------------------------------------
    for (int i = tid; i < 1 + T.n_par; i += NT) V[i] = (i == 0) ? 1.0 : par[i - 1];
    __syncthreads();
    for (int l = 0; l < T.n_levels; ++l) {
      for (int e = T.level_ptr[l] + tid; e < T.level_ptr[l + 1]; e += NT) {
        double acc = 0.0;
        for (int t = T.tape_ptr[e]; t < T.tape_ptr[e + 1]; ++t) {
          const int4 f = __ldg(reinterpret_cast<const int4*>(T.tape_fac) + t);
          acc += T.tape_coef[t] * V[f.x] * V[f.y] * V[f.z] * V[f.w];
        }
        switch (T.tape_func[e]) {
          case 1: acc = 1.0 / acc; break;
          case 2: acc = (acc >= 0.0) ? 1.0 : 0.0; break;
          case 3: acc = (acc > 0.0) ? 1.0 : 0.0; break;
          case 4: acc = sin(acc); break;
          case 5: acc = cos(acc); break;
          case 6: acc = sqrt(acc); break;
          default: break;
        }
        V[1 + T.n_par + e] = acc;
      }
      __syncthreads();
    }
    // ---- S2: x ------------------------------------------------------------------
    for (int i = tid; i <= n; i += NT) { xe[i] = (i < n) ? x0[i] : 1.0; xt[i] = 1.0; }
    __syncthreads();
    if (XL) {
      for (int l = tid; l < T.n_mid; l += NT) { const int2 r = T.midg[l]; xe[n + 1 + l] = eval_range(T.Gt, r.x, r.y, V, xe); }
      __syncthreads();
      jac_xl(T, V, xe, jx, jval, nullptr, true);
    }

    // ---- S3: row classification, scaling, starting point -----------------------
    double fmaxv = 0.0;
    for (int j = tid; j < n; j += NT)
      fmaxv = fmax(fmaxv, fabs(eval_range(T.DFt, T.dfptr[j], T.dfptr[j + 1], V, xe)));
    {
      double r1[1] = {fmaxv};
      block_reduce<OP_MAX>(r1, red);
      fmaxv = r1[0];
    }
    const double smg = O.scaling_max_gradient;
    const double fsc = (fmaxv > smg) ? fmax(smg / fmaxv, 1e-8) : 1.0;
    for (int i = tid; i < m; i += NT) {
      const RowRec rr = T.rowrec[i];
      // Jacobian row: max |J| for the gradient-based scaling
      double gm = 0.0;
      if (XL) {       // jval = unscaled Jacobian (jac_xl)
        for (int k = 0; k < rr.ns; ++k) gm = fmax(gm, fabs(jval[rr.s0 + k]));
      } else {
        double acc = 0.0; int cur = 0, aux;
        for (int k = rr.jt0; k < rr.jt1; ++k) {
          const double v = term_value(T.Jt + k, V, xe, &aux);
          if (aux != cur) { gm = fmax(gm, fabs(acc)); acc = 0.0; cur = aux; }
          acc += v;
        }
        gm = fmax(gm, fabs(acc));
      }
      const double d = (gm > smg) ? fmax(smg / gm, 1e-8) : 1.0;
      dsc[i] = d;
      const double lb = lbg[i], ub = ubg[i];
      const bool eq = (lb == ub);
      const bool hL = (lb > -INF_BOUND) && !eq, hU = (ub < INF_BOUND) && !eq;
      rt[i] = (unsigned char)((hL ? 1 : 0) | (hU ? 2 : 0) | (eq ? 4 : 0));
      double l = lb * d, uu = ub * d;
      beq[i] = l;
      if (hL) l -= O.bound_relax_factor * fmax(1.0, fabs(l));
      if (hU) uu += O.bound_relax_factor * fmax(1.0, fabs(uu));
      sL[i] = l; sU[i] = uu;
      const double gi = d * eval_range(T.Gt, rr.g0, rr.g1, V, xe);
      g[i] = gi;
      double si = gi;
      const double k1 = O.bound_push, k2 = O.bound_frac;
      double pl = k1 * fmax(1.0, fabs(l)), pu = k1 * fmax(1.0, fabs(uu));
      if (hL && hU) { pl = fmin(pl, k2 * (uu - l)); pu = fmin(pu, k2 * (uu - l)); }
      if (hL) si = fmax(si, l + pl);
      if (hU) si = fmin(si, uu - pu);
      s[i] = si;
      double yi = 0.0;
      if (A.lam0) yi = A.lam0[(size_t)inst * m + i] * fsc / d;
      y[i] = yi;
      zL[i] = hL ? fmax(O.mult_bound_push, -yi) : 0.0;
      zU[i] = hU ? fmax(O.mult_bound_push, yi) : 0.0;
    }
    __syncthreads();
    if (tid == 0) {
      int ne = 0, nbnd = 0, bad = 0;
      for (int i = 0; i < m; ++i) {
        const int r = rt[i];
        if (r & 4) {
          if (ne < T.n_eq && T.eq_rows[ne] == i) { eqrow[ne] = i; eqidx[i] = ne; } else bad = 1;
          ++ne;
        } else eqidx[i] = -1;
        nbnd += (r & 1) + ((r >> 1) & 1);
      }
      if (ne != T.n_eq) bad = 1;
      ctl.n_eq = bad ? -1 : ne; ctl.n_bounds = nbnd;
      ctl.mu = O.mu_init; ctl.tau = fmax(TAU_MIN, 1.0 - O.mu_init);
      ctl.theta_max = -1.0; ctl.theta_min = -1.0;
      ctl.delta_w_last = 0.0; ctl.nfilt = 0; ctl.status = -1; ctl.iter = 0;
      ctl.fsc = fsc; ctl.alpha = 0.0; ctl.delta_w = 0.0; ctl.n_restart = 0;
      ctl.f = fsc * eval_range(T.Ft, 0, T.n_f, V, xe);
    }
    __syncthreads();
    if (ctl.n_eq < 0) {   // equality pattern differs from the lowered structure
      if (tid == 0) { A.status[inst] = OMG_ERROR_IN_STEP_COMPUTATION; A.iters[inst] = 0; A.f[inst] = 0.0; }
      for (int i = tid; i < n; i += NT) A.x[(size_t)inst * n + i] = x0[i];
      for (int i = tid; i < m; i += NT) A.lam[(size_t)inst * m + i] = 0.0;
      __syncthreads();
      continue;
    }
    const int n_eq = ctl.n_eq;
    const int N = T.N;
    const int n_bounds = ctl.n_bounds;

    // =========================== IP iterations ===============================
    for (int iter = 0;; ++iter) {
      TICK(0);   // setup / previous accept
      // ---- I1: rows: Jacobian values, residual terms (g kept from the trial) ------
      double rv[NRED];
      // 0 cinf(max) 1 maxprod(max) 2 minprod(min) 3 viol(max) 4 rsinf(max)
      // 5 rsinf_un(max) 6 ysum 7 zsum 8 theta 9 logsum 10 rxinf(max)   (NRED_OPS)
      for (int r = 0; r < NRED; ++r) rv[r] = 0.0;
      rv[2] = 1e300;
      if (XL) jac_xl(T, V, xe, jx, jval, dsc, false);
      for (int i = tid; i < m; i += NT) {
        const RowRec rr = T.rowrec[i];
        const int r = rt[i];
        const double d = dsc[i];
        if (!XL) {
          double acc = 0.0; int cur = 0, aux;
          double* jv = jval + rr.s0;
#pragma unroll 4
          for (int k = rr.jt0; k < rr.jt1; ++k) {
            const double v = term_value(T.Jt + k, V, xe, &aux);
            if (aux != cur) { jv[cur] = d * acc; acc = 0.0; cur = aux; }
            acc += v;
          }
          if (rr.ns > 0) jv[cur] = d * acc;
        }
        const double gi = g[i], si = s[i], yi = y[i];
        const double ci = (r & 4) ? gi - beq[i] : gi - si;
        rv[0] = fmax(rv[0], fabs(ci));
        rv[8] += fabs(ci);
        double zl = 0.0, zu = 0.0;
        if (r & 1) { zl = zL[i]; const double dl = si - sL[i]; const double pz = dl * zl;
          rv[1] = fmax(rv[1], pz); rv[2] = fmin(rv[2], pz); rv[9] += log(dl); rv[7] += zl; }
        if (r & 2) { zu = zU[i]; const double du = sU[i] - si; const double pz = du * zu;
          rv[1] = fmax(rv[1], pz); rv[2] = fmin(rv[2], pz); rv[9] += log(du); rv[7] += zu; }
        const double gun = gi / d;
        if (r & 6) rv[3] = fmax(rv[3], gun - ubg[i]);
        if (r & 5) rv[3] = fmax(rv[3], lbg[i] - gun);
        if (!(r & 4)) { const double rs = fabs(-yi - zl + zu);
          rv[4] = fmax(rv[4], rs); rv[5] = fmax(rv[5], rs * d); }
        rv[6] += fabs(yi);
      }
      __syncthreads();   // jval visible to the column pass
      TICK(1);   // row pass
      // ---- I2: columns: grad f, dual residual ------------------------------------
      for (int j = tid; j < n; j += NT) {
        const double gj = ctl.fsc * eval_range(T.DFt, T.dfptr[j], T.dfptr[j + 1], V, xe);
        gf[j] = gj;
        double rx = gj;
        const int q0 = T.colptr[j], q1 = T.colptr[j + 1];
#pragma unroll 4
        for (int q = q0; q < q1; ++q) {
          const unsigned cr = __ldg(T.colrec + q);
          rx += jval[cr & 0xffffu] * y[cr >> 16];
        }
        rv[10] = fmax(rv[10], fabs(rx));
      }
      block_reduce<NRED_OPS>(rv, red);
      const double cinf = rv[0], maxprod = rv[1], minprod = rv[2], viol = rv[3];
      const double dinf = fmax(rv[10], rv[4]);
      const double dinf_un = fmax(rv[10], rv[5]) / ctl.fsc;
      const double ysum = rv[6], zsum = rv[7], theta = rv[8], logsum = rv[9];
      const double s_d = fmax(S_MAX, (ysum + zsum) / fmax(1.0, (double)(m + n_bounds))) / S_MAX;
      const double s_c = fmax(S_MAX, zsum / fmax(1.0, (double)n_bounds)) / S_MAX;
      double mu = ctl.mu;
      const double cmpl0 = n_bounds ? fmax(fabs(maxprod), fabs(minprod)) : 0.0;
      const double E0 = fmax(fmax(dinf / s_d, cinf), cmpl0 / s_c);
      TICK(2);   // column pass + reduction
      // ---- I3: termination + barrier update (uniform) ---------------------------
      int status = -1;
      if (!isfinite(E0) || !isfinite(theta)) status = OMG_INVALID_NUMBER_DETECTED;
      else if (E0 <= O.tol && dinf_un <= O.dual_inf_tol && viol <= O.constr_viol_tol &&
               cmpl0 / ctl.fsc <= O.compl_inf_tol) status = OMG_SOLVE_SUCCEEDED;
      else if (iter >= O.max_iter) status = OMG_MAX_ITER_EXCEEDED;
      if (tracing && tid == 0 && iter < TRACE_ROWS - 2) {
        double* tr = A.trace + iter * TRACE_COLS;
        tr[0] = iter; tr[1] = ctl.f / ctl.fsc; tr[2] = cinf; tr[3] = dinf; tr[4] = mu; tr[5] = E0;
        tr[6] = ctl.alpha; tr[7] = ctl.delta_w;
      }
      if (status >= 0) { if (tid == 0) { ctl.status = status; ctl.iter = iter; } break; }
      {
        const double mu_min = fmin(O.tol, O.compl_inf_tol * ctl.fsc) / (KAPPA_EPS + 1.0);
        bool changed = false;
        for (;;) {
          const double cm = n_bounds ? fmax(fabs(maxprod - mu), fabs(minprod - mu)) : 0.0;
          const double Emu = fmax(fmax(dinf / s_d, cinf), cm / s_c);
          if (Emu <= KAPPA_EPS * mu && mu > mu_min) {
            mu = fmax(mu_min, fmin(KAPPA_MU * mu, pow(mu, THETA_MU)));
            changed = true;
          } else break;
        }
        __syncthreads();
        if (tid == 0) {
          ctl.mu = mu; ctl.tau = fmax(TAU_MIN, 1.0 - mu);
          if (changed) ctl.nfilt = 0;
          if (ctl.theta_max < 0.0) {
            ctl.theta_max = THETA_MAX_FACT * fmax(1.0, theta);
            ctl.theta_min = THETA_MIN_FACT * fmax(1.0, theta);
          }
          ctl.theta = theta;
          ctl.phi = ctl.f - mu * logsum;
          ctl.delta_w = 0.0; ctl.delta_c = 0.0; ctl.first_try = 1;
        }
      }
      __syncthreads();
      const double tau = ctl.tau;
      TICK(3);   // barrier logic
      // ---- I4: Sigma, w = Sigma r_d + phi_s, sigma-scaled Jacobian ----------------
      for (int i = tid; i < m; i += NT) {
        const int r = rt[i];
        double sg = 0.0, ph = 0.0, rd = 0.0;
        if (!(r & 4)) {
          const double si = s[i];
          rd = g[i] - si;
          if (r & 1) { const double dl = si - sL[i]; sg += zL[i] / dl; ph -= mu / dl; }
          if (r & 2) { const double du = sU[i] - si; sg += zU[i] / du; ph += mu / du; }
        }
        sig[i] = sg;
        wv[i] = (r & 4) ? y[i] : (sg * rd + ph);
        const RowRec rr = T.rowrec[i];
        for (int k = 0; k < rr.ns; ++k) jsv[rr.s0 + k] = sg * jval[rr.s0 + k];
      }
      __syncthreads();
      TICK(4);   // sigma pass

      if (XL) {   // multipliers of the mids' Hessians: mu = A^T (y*dsc), A raw (unscaled)
        for (int l = tid; l < T.n_mid; l += NT) {
          double acc = 0.0;
          for (int e = T.mu_ptr[l]; e < T.mu_ptr[l + 1]; ++e) {
            const int i = T.mu_row[e];
            acc += y[i] * dsc[i] * jx[T.mu_slot[e]];
          }
          mu_mid[l] = acc;
        }
        __syncthreads();
      }
      // ---- I7/I8: assemble + factorise, with inertia correction -----------------
      bool assembled = false;   // the assembled K (delta = 0) is kept in scratch for the retries
      for (;;) {
        if (assembled) {
          const double2* C2 = reinterpret_cast<const double2*>(Kc);
          double2* K2 = reinterpret_cast<double2*>(K);
          const int h2 = (T.env_size + 1) >> 1;
          for (int q = tid; q < h2; q += NT) K2[q] = C2[q];
          __syncthreads();
          for (int j = tid; j < n; j += NT) {
            const int pj = T.pos_var[j];
            const double v = K[T.kdiag[pj]] + ctl.delta_w;
            K[T.kdiag[pj]] = v; diag0[pj] = fabs(v);
          }
          for (int k = tid; k < n_eq; k += NT) {
            const int pk = T.pos_eq[k];
            K[T.kdiag[pk]] = -ctl.delta_c; diag0[pk] = ctl.delta_c;
          }
          if (tid == 0) { ctl.fail = 0; ctl.eq_fail = 0; }
          __syncthreads();
        } else {
        {
          double2* K2 = reinterpret_cast<double2*>(K);
          const int h2 = (T.env_size + 1) >> 1;
          for (int q = tid; q < h2; q += NT) K2[q] = make_double2(0.0, 0.0);
        }
        __syncthreads();
        // H positions: gather J^T Sigma J (+ delta_w on the diagonal)
        for (int q = tid; q < T.nnz_h; q += NT) {
          const HqRec h = T.hq[q];
          double acc = 0.0;
#pragma unroll 4
          for (int e = h.p0; e < h.p1; ++e) {
            const unsigned pk = __ldg(T.hpack + e);
            acc += jsv[pk & 0xffffu] * jval[pk >> 16];
          }
          if (h.diag) acc += ctl.delta_w;
          K[h.dst] = acc;
        }
        __syncthreads();
        TICK(5);   // zero + H gather
        // Lagrangian Hessian W (lambda = y*dsc, objective factor fsc)
        if (XL) {   // slots differ widely in term count: one warp per slot
          const int lane = tid & 31;
          for (int q = tid >> 5; q < T.nnz_w + T.nnz_wx; q += NWARP) {
            const WRec w = T.wrec[q];
            double acc = 0.0;
            for (int t = w.t0 + lane; t < w.t1; t += 32) {
              int lr;
              double v = term_value(T.Wt + t, V, xe, &lr);
              v *= (lr < m) ? (y[lr] * dsc[lr]) : (lr == m ? ctl.fsc : mu_mid[lr - m - 1]);
              acc += v;
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) acc += __shfl_down_sync(FULL, acc, o);
            if (lane == 0) { if (q < T.nnz_w) K[w.dst] += acc; else wx[w.dst] = acc; }
          }
          if (T.nnz_wx) {   // X^T C + C^T X + C^T M C, one thread per H position (deterministic)
            __syncthreads();
            for (int e = tid; e < T.n_xq; e += NT) {
              const HqRec h = T.xq[e];
              double acc = 0.0;
              for (int r = h.p0; r < h.p1; ++r) {
                const int4 pr = T.xqp[r];
                const double v = wx[pr.x] * jx[pr.y];
                acc += (pr.z >= 0) ? v * jx[pr.z] : v;
              }
              K[h.dst] += acc;
            }
          }
        } else
        for (int q = tid; q < T.nnz_w; q += NT) {
          const WRec w = T.wrec[q];
          double acc = 0.0;
          for (int t = w.t0; t < w.t1; ++t) {
            int lr;
            double v = term_value(T.Wt + t, V, xe, &lr);
            v *= (lr < m) ? (y[lr] * dsc[lr]) : ctl.fsc;
            acc += v;
          }
          K[w.dst] += acc;
        }
        __syncthreads();
        for (int j = tid; j < n; j += NT) {
          const int pj = T.pos_var[j];
          diag0[pj] = fabs(K[T.kdiag[pj]]);
        }
        // equality border + right-hand-side row
        const int rhs0 = KS_EPTR[N];
        for (int k = tid; k < n_eq; k += NT) {
          const int i = eqrow[k], pk = T.pos_eq[k];
          const RowRec rr = T.rowrec[i];
          for (int q = 0; q < rr.ns; ++q) K[T.jdst[rr.s0 + q]] = jval[rr.s0 + q];
          K[T.kdiag[pk]] = -ctl.delta_c;
          diag0[pk] = ctl.delta_c;
          K[rhs0 + pk] = -(g[i] - beq[i]);
        }
        for (int j = tid; j < n; j += NT) {
          double acc = gf[j];
          const int q0 = T.colptr[j], q1 = T.colptr[j + 1];
#pragma unroll 4
          for (int q = q0; q < q1; ++q) {
            const unsigned cr = __ldg(T.colrec + q);
            acc += jval[cr & 0xffffu] * wv[cr >> 16];
          }
          K[rhs0 + T.pos_var[j]] = -acc;
        }
        if (tid == 0) { ctl.fail = 0; ctl.eq_fail = 0; }
        __syncthreads();
        {
          double2* C2 = reinterpret_cast<double2*>(Kc);
          const double2* K2 = reinterpret_cast<const double2*>(K);
          const int h2 = (T.env_size + 1) >> 1;
          for (int q = tid; q < h2; q += NT) C2[q] = K2[q];
          assembled = true;
        }
        }
        TICK(6);   // W + border + rhs
        factor_env<WIDE>(T, S, K, &ctl, tracing ? phase_cyc : nullptr, O.inertia_mode);
        __syncthreads();
        phase_t0 = clock64();
        if (!ctl.fail) break;
        // inertia correction (IPOPT algorithm IC on the condensed matrix)
        if (tid == 0) {
          if (ctl.eq_fail) ctl.delta_c = DELTA_C_VAL * pow(mu, DELTA_C_EXP);
          if (ctl.first_try) {
            ctl.delta_w = (ctl.delta_w_last == 0.0) ? DELTA_W0
                          : fmax(DELTA_W_MIN, KAPPA_W_MINUS * ctl.delta_w_last);
            ctl.first_try = 0;
          } else {
            ctl.delta_w *= (ctl.delta_w_last == 0.0) ? KAPPA_W_PLUS_FIRST : KAPPA_W_PLUS;
          }
        }
        __syncthreads();
        if (ctl.delta_w > DELTA_W_MAX) break;
      }
      if (ctl.fail) {
        if (tid == 0) { ctl.status = OMG_ERROR_IN_STEP_COMPUTATION; ctl.iter = iter; }
        __syncthreads();
        break;
      }
      if (tid == 0 && ctl.delta_w > 0.0) ctl.delta_w_last = ctl.delta_w;
      // ---- I9: solve -----------------------------------------------------------
      for (int j = tid; j < N; j += NT) u[j] = K[KS_EPTR[N] + j];
      __syncthreads();
      back_solve_env(T, S, K);
      for (int j = tid; j < n; j += NT) dx[j] = u[T.pos_var[j]];
      for (int k = tid; k < n_eq; k += NT) dx[n + k] = u[T.pos_eq[k]];
      __syncthreads();
      TICK(10);  // back substitution
      // ---- I10: ds, dy, dz, fraction to the boundary --------------------------
      double sv[4];   // 0 a_p(min) 1 a_d(min) 2 gphi(sum)
      sv[0] = 1.0; sv[1] = 1.0; sv[2] = 0.0; sv[3] = 0.0;
      for (int i = tid; i < m; i += NT) {
        const int r = rt[i];
        const RowRec rr = T.rowrec[i];
        double jd = 0.0;
#pragma unroll 4
        for (int k = 0; k < rr.ns; ++k) jd += jval[rr.s0 + k] * dx[T.jcol16[rr.s0 + k]];
        if (r & 4) {
          ds[i] = 0.0; dy[i] = dx[n + eqidx[i]]; dzL[i] = 0.0; dzU[i] = 0.0;
        } else {
          const double si = s[i];
          const double dsi = jd + (g[i] - si);
          double ph = 0.0, a = 0.0, b = 0.0;
          if (r & 1) { const double dl = si - sL[i]; const double z = zL[i]; ph -= mu / dl;
            a = mu / dl - z - (z / dl) * dsi;
            if (dsi < 0.0) sv[0] = fmin(sv[0], -tau * dl / dsi);
            if (a < 0.0) sv[1] = fmin(sv[1], -tau * z / a); dzL[i] = a; }
          if (r & 2) { const double du = sU[i] - si; const double z = zU[i]; ph += mu / du;
            b = mu / du - z + (z / du) * dsi;
            if (dsi > 0.0) sv[0] = fmin(sv[0], tau * du / dsi);
            if (b < 0.0) sv[1] = fmin(sv[1], -tau * z / b); }
          ds[i] = dsi; dzU[i] = b;
          dy[i] = sig[i] * dsi + ph - y[i];
          sv[2] += ph * dsi;
        }
      }
      for (int j = tid; j < n; j += NT) sv[2] += gf[j] * dx[j];
      block_reduce<OP_MIN, OP_MIN, OP_SUM, OP_SUM>(sv, red);
      const double a_p = sv[0], a_d = sv[1], gphi = sv[2];
      TICK(11);  // step pass
      // ---- I11: filter line search --------------------------------------------
      const double theta0 = ctl.theta, phi0 = ctl.phi;
      double a_min;
      if (gphi < 0.0) {
        a_min = fmin(GAMMA_THETA, GAMMA_PHI * theta0 / (-gphi));
        if (theta0 <= ctl.theta_min)
          a_min = fmin(a_min, DELTA_LS * pow(theta0, S_THETA) / pow(-gphi, S_PHI));
      } else a_min = GAMMA_THETA;
      a_min *= GAMMA_ALPHA;
      double alpha = a_p;
      bool accepted = false, ftype = false;
      double ft = 0.0;
      int n_ls = 0;
      while (alpha >= a_min && n_ls < MAX_LS) {
        ++n_ls;
        for (int j = tid; j < n; j += NT) xt[j] = xe[j] + alpha * dx[j];
        __syncthreads();
        if (XL) {
          for (int l = tid; l < T.n_mid; l += NT) { const int2 r = T.midg[l]; xt[n + 1 + l] = eval_range(T.Gt, r.x, r.y, V, xt); }
          __syncthreads();
        }
        double tv[3];  // 0 theta 1 logsum 2 f
        tv[0] = 0.0; tv[1] = 0.0; tv[2] = 0.0;
        for (int i = tid; i < m; i += NT) {
          const RowRec rr = T.rowrec[i];
          const int r = rt[i];
          const double gi = dsc[i] * eval_range(T.Gt, rr.g0, rr.g1, V, xt);
          gt[i] = gi;
          if (r & 4) tv[0] += fabs(gi - beq[i]);
          else {
            const double si = s[i] + alpha * ds[i];
            st[i] = si;
            tv[0] += fabs(gi - si);
            if (r & 1) tv[1] += log(si - sL[i]);
            if (r & 2) tv[1] += log(sU[i] - si);
          }
        }
        // objective terms spread over the block (summed by the same reduction)
        for (int t = tid; t < T.n_f; t += NT) { int aux; tv[2] += term_value(T.Ft + t, V, xt, &aux); }
        block_reduce<OP_SUM, OP_SUM, OP_SUM>(tv, red);
        ft = ctl.fsc * tv[2];
        const double tht = tv[0], pht = ft - mu * tv[1];
        bool ok = isfinite(pht) && isfinite(tht) && tht <= ctl.theta_max;
        if (ok) {
          const int nf = ctl.nfilt;
          for (int q = 0; q < nf; ++q)
            if (!(tht < filt[2 * q] || pht < filt[2 * q + 1])) { ok = false; break; }
        }
        ftype = false;
        if (ok) {
          const bool switching = (theta0 <= ctl.theta_min && gphi < 0.0 &&
                                  alpha * pow(-gphi, S_PHI) > DELTA_LS * pow(theta0, S_THETA));
          if (switching) { ok = cmp_le(pht - phi0, ETA_PHI * alpha * gphi, phi0); ftype = ok; }
          else ok = cmp_le(tht, (1.0 - GAMMA_THETA) * theta0, theta0) ||
                    cmp_le(pht - phi0, -GAMMA_PHI * theta0, phi0);
        }
        if (ok) { accepted = true; break; }
        alpha *= 0.5;
      }
      bool soft = false;
      if (!accepted && O.soft_resto) {
        // ---- soft restoration (IPOPT): the filter rejected every trial step; accept a step
        // along the same direction if it reduces the primal-dual error of the barrier problem
        __syncthreads();
        double pv[1];
        pv[0] = 0.0;
        for (int i = tid; i < m; i += NT) {
          const int r = rt[i];
          if (r & 4) { pv[0] += fabs(g[i] - beq[i]); continue; }
          const double si = s[i];
          double zl = 0.0, zu = 0.0, acc = fabs(g[i] - si);
          if (r & 1) { zl = zL[i]; acc += fabs((si - sL[i]) * zl - mu); }
          if (r & 2) { zu = zU[i]; acc += fabs((sU[i] - si) * zu - mu); }
          pv[0] += acc + fabs(-y[i] - zl + zu);
        }
        for (int j = tid; j < n; j += NT) {
          double rx = gf[j];
          for (int q = T.colptr[j]; q < T.colptr[j + 1]; ++q) {
            const unsigned cr = __ldg(T.colrec + q);
            rx += jval[cr & 0xffffu] * y[cr >> 16];
          }
          pv[0] += fabs(rx);
        }
        block_reduce<OP_SUM>(pv, red);
        const double pd0 = pv[0];
        alpha = a_p;
        for (int n_try = 0; n_try < 12; ++n_try) {
          for (int j = tid; j < n; j += NT) xt[j] = xe[j] + alpha * dx[j];
          __syncthreads();
          if (XL) {
            for (int l = tid; l < T.n_mid; l += NT) { const int2 r = T.midg[l]; xt[n + 1 + l] = eval_range(T.Gt, r.x, r.y, V, xt); }
            __syncthreads();
            jac_xl(T, V, xt, jx, jsv, dsc, false);       // trial Jacobian -> jsv (free until the next sigma pass)
          }
          const double az = fmin(alpha, a_d);
          pv[0] = 0.0;
          for (int i = tid; i < m; i += NT) {
            const RowRec rr = T.rowrec[i];
            const int r = rt[i];
            const double d = dsc[i];
            if (!XL) {
              double acc = 0.0; int cur = 0, aux;
              double* jv = jsv + rr.s0;
              for (int k = rr.jt0; k < rr.jt1; ++k) {
                const double v = term_value(T.Jt + k, V, xt, &aux);
                if (aux != cur) { jv[cur] = d * acc; acc = 0.0; cur = aux; }
                acc += v;
              }
              if (rr.ns > 0) jv[cur] = d * acc;
            }
            const double gi = d * eval_range(T.Gt, rr.g0, rr.g1, V, xt);
            gt[i] = gi;
            const double yt = y[i] + alpha * dy[i];
            wv[i] = yt;
            if (r & 4) { pv[0] += fabs(gi - beq[i]); continue; }
            const double si = s[i] + alpha * ds[i];
            st[i] = si;
            double zl = 0.0, zu = 0.0, acc = fabs(gi - si);
            if (r & 1) { zl = zL[i] + az * dzL[i]; acc += fabs((si - sL[i]) * zl - mu); }
            if (r & 2) { zu = zU[i] + az * dzU[i]; acc += fabs((sU[i] - si) * zu - mu); }
            pv[0] += acc + fabs(-yt - zl + zu);
          }
          __syncthreads();
          for (int j = tid; j < n; j += NT) {
            double rx = ctl.fsc * eval_range(T.DFt, T.dfptr[j], T.dfptr[j + 1], V, xt);
            for (int q = T.colptr[j]; q < T.colptr[j + 1]; ++q) {
              const unsigned cr = __ldg(T.colrec + q);
              rx += jsv[cr & 0xffffu] * wv[cr >> 16];
            }
            pv[0] += fabs(rx);
          }
          block_reduce<OP_SUM>(pv, red);
          if (isfinite(pv[0]) && pv[0] <= SOFT_RESTO_FACTOR * pd0) {
            double fv[1]; fv[0] = 0.0;
            for (int t = tid; t < T.n_f; t += NT) { int aux; fv[0] += term_value(T.Ft + t, V, xt, &aux); }
            block_reduce<OP_SUM>(fv, red);
            ft = ctl.fsc * fv[0];
            accepted = true; soft = true; ftype = true;
            break;
          }
          alpha *= 0.5;
        }
      }
      if (!accepted) {
        if (ctl.n_restart < O.max_restarts) {
          // feasibility restart (stand-in for IPOPT's restoration phase, oracle/ipm_ref.py):
          // keep x, re-centre the slacks, zero the multipliers, clear the filter, mu = restart_mu
          __syncthreads();
          const double mu_r = O.restart_mu;
          for (int i = tid; i < m; i += NT) {
            const int r = rt[i];
            double si = g[i];
            if (r & 1) si = fmax(si, sL[i] + O.restart_push * fmax(1.0, fabs(sL[i])));
            if (r & 2) si = fmin(si, sU[i] - O.restart_push * fmax(1.0, fabs(sU[i])));
            s[i] = si; y[i] = 0.0;
            if (r & 1) zL[i] = mu_r / (si - sL[i]);
            if (r & 2) zU[i] = mu_r / (sU[i] - si);
          }
          if (tid == 0) {
            ctl.n_restart += 1; ctl.mu = mu_r; ctl.tau = fmax(TAU_MIN, 1.0 - mu_r);
            ctl.nfilt = 0; ctl.theta_max = -1.0; ctl.delta_w_last = 0.0;
          }
          __syncthreads();
          continue;
        }
        if (tid == 0) { ctl.status = OMG_RESTORATION_FAILED; ctl.iter = iter; }
        __syncthreads();
        break;
      }
      __syncthreads();
      if (tid == 0) {
        if (soft) ctl.nfilt = 0;
        if (!ftype) {        // augment the filter, dropping dominated entries
          const double th = (1.0 - GAMMA_THETA) * theta0, ph = phi0 - GAMMA_PHI * theta0;
          int nf = 0;
          for (int q = 0; q < ctl.nfilt; ++q)
            if (!(filt[2 * q] >= th && filt[2 * q + 1] >= ph)) {
              filt[2 * nf] = filt[2 * q]; filt[2 * nf + 1] = filt[2 * q + 1]; ++nf; }
          if (nf >= MAXF) {
            for (int q = 1; q < nf; ++q) { filt[2 * (q - 1)] = filt[2 * q]; filt[2 * (q - 1) + 1] = filt[2 * q + 1]; }
            --nf;
          }
          filt[2 * nf] = th; filt[2 * nf + 1] = ph; ++nf;
          ctl.nfilt = nf;
        }
        ctl.f = ft; ctl.alpha = alpha;
      }
      TICK(12);  // line search
      // ---- I12: accept -------------------------------------------------------------
      for (int j = tid; j < n_xe; j += NT) xe[j] = xt[j];
      for (int i = tid; i < m; i += NT) {
        const int r = rt[i];
        g[i] = gt[i];
        y[i] += alpha * dy[i];
        if (!(r & 4)) {
          const double si = st[i];
          s[i] = si;
          if (r & 1) { const double dl = si - sL[i]; double z = zL[i] + a_d * dzL[i];
            z = fmin(fmax(z, mu / (KAPPA_SIGMA * dl)), KAPPA_SIGMA * mu / dl); zL[i] = z; }
          if (r & 2) { const double du = sU[i] - si; double z = zU[i] + a_d * dzU[i];
            z = fmin(fmax(z, mu / (KAPPA_SIGMA * du)), KAPPA_SIGMA * mu / du); zU[i] = z; }
        }
      }
      __syncthreads();
    }  // iterations

    // ---- write results -----------------------------------------------------------
    __syncthreads();
    for (int i = tid; i < n; i += NT) A.x[(size_t)inst * n + i] = xe[i];
    for (int i = tid; i < m; i += NT) A.lam[(size_t)inst * m + i] = y[i] * dsc[i] / ctl.fsc;
    if (tracing && tid == 0) {
      TICK(13);
      double* tr = A.trace + (TRACE_ROWS - 2) * TRACE_COLS;
      for (int k = 0; k < NPHASE; ++k) tr[k] = phase_cyc[k];
    }
    if (tid == 0) {
      A.f[inst] = ctl.f / ctl.fsc;
      A.status[inst] = ctl.status;
      A.iters[inst] = ctl.iter;
    }
    __syncthreads();
  }
}

template <bool WIDE> __global__ void __launch_bounds__(512, 1)
omg_ipm_kernel(const DevTab T, const omg_options O, const Batch A, const Smem S) { ipm_body<false, WIDE>(T, O, A, S); }

// sparse variant (omg_sp.cuh): L D L^T on the minimum-degree structure, thread streams, 128 or
// 256 threads per instance, as many blocks per SM as shared memory allows (config 2: 3)
#include "omg_sp.cuh"
// (__grid_constant__: the out-of-line parts take the parameters by reference without a local copy)
__global__ void __launch_bounds__(128, 4)
omg_ipm_kernel_sp(const __grid_constant__ DevTab T, const __grid_constant__ SpTab P, const __grid_constant__ omg_options O,
                  const __grid_constant__ Batch A, const __grid_constant__ SpSmem S) {
  ipm_body_sp(T, P, O, A, S);
}

template <bool WIDE> __global__ void __launch_bounds__(256, 2)
omg_ipm_kernel_2cta(const DevTab T, const omg_options O, const Batch A, const Smem S) { ipm_body<false, WIDE>(T, O, A, S); }

template <bool WIDE> __global__ void __launch_bounds__(512, 1)
omg_ipm_kernel_xl(const DevTab T, const omg_options O, const Batch A, const Smem S) { ipm_body<true, WIDE>(T, O, A, S); }

// XL with K in scratch: the block needs little shared memory, and the kernel is bound by the
// latency of its L2 streams, so two blocks per SM overlap better than one wide block
template <bool WIDE> __global__ void __launch_bounds__(256, 2)
omg_ipm_kernel_xl_2cta(const DevTab T, const omg_options O, const Batch A, const Smem S) { ipm_body<true, WIDE>(T, O, A, S); }

// one shift block (offset off, basis length L, nc columns) of one instance, spread over the threads
// of a block: dst[off + c*L + i] = sum_k T[i,k] src[off + c*L + k] (src must not alias dst)
__device__ __forceinline__ void omg_shift_block(const double* Tb, const double* src, double* dst, int off, int L,
                                                int nc) {
  for (int e = threadIdx.x; e < L * nc; e += blockDim.x) {
    const int c = e / L, i = e % L;
    double acc = 0.0;
    for (int k = 0; k < L; ++k) acc += Tb[i * L + k] * src[off + c * L + k];
    dst[off + c * L + i] = acc;
  }
}

// warm-start shift: x[b, off + c*len + i] <- sum_k T[i,k] x[b, off + c*len + k]
__global__ void omg_shift_kernel(double* x, int B, int n, int n_blocks, const int* offs,
                                 const int* lens, const int* ncols, const int* toffs,
                                 const double* Tm) {
  OMG_DYN_SHARED(xs);
  const int b = blockIdx.x;
  if (b >= B) return;
  double* xb = x + (size_t)b * n;
  for (int i = threadIdx.x; i < n; i += blockDim.x) xs[i] = xb[i];
  __syncthreads();
  for (int blk = 0; blk < n_blocks; ++blk) {
    const int L = lens[blk], nc = ncols[blk], off = offs[blk];
    const double* Tb = Tm + toffs[blk];
    omg_shift_block(Tb, xs, xb, off, L, nc);
  }
}

// vehicle models for the batched state prediction and the closed-loop plant step (reference
// Vehicle.ode and splines2signals of each class)
enum { OMG_ODE_INTEGRATOR = 0, OMG_ODE_QUADROTOR3D = 1, OMG_ODE_QUADROTOR2D = 2, OMG_ODE_DUBINS = 3,
       OMG_ODE_HOLONOMIC_ORIENT = 4, OMG_ODE_SIMPLE_QUADROTOR3D = 5, OMG_ODE_N_MODELS = 6 };
#define OMG_ODE_MAX_STATE 8

// Per model: state and input sizes (0: any, with n_state = n_input), the rows of spline
// derivatives its planned input reads (value and first derivative = 2; the input splines are
// its first n_input spline columns), and the right-hand side it integrates.
struct OmgOdeModel { int n_state, n_input, n_der, ode; };
static const OmgOdeModel omg_ode_models[OMG_ODE_N_MODELS] = {
  {0, 0, 2, OMG_ODE_INTEGRATOR},      // Holonomic, Holonomic1D, Holonomic3D
  {8, 3, 2, OMG_ODE_QUADROTOR3D},     // Quadrotor3D
  {5, 2, 4, OMG_ODE_QUADROTOR2D},     // Quadrotor
  {3, 2, 2, OMG_ODE_DUBINS},          // Dubins
  {3, 3, 2, OMG_ODE_INTEGRATOR},      // HolonomicOrient: (x, y, theta)' = input
  {8, 3, 4, OMG_ODE_QUADROTOR3D},     // SimpleQuadrotor3D: Quadrotor3D's state and ODE
};

static bool omg_ode_sizes_ok(int model, int n_state, int n_input) {
  const OmgOdeModel& m = omg_ode_models[model];
  return m.n_state ? (n_state == m.n_state && n_input == m.n_input) : (n_state == n_input && n_input >= 1);
}

__device__ __forceinline__ void ode_rhs(int ode, int ns, const double* st, const double* u, double* d) {
  if (ode == OMG_ODE_QUADROTOR3D) {            // quadrotor3d.py:308-312, quadrotor3d_simple.py:186-190
    const double phi = st[6], theta = st[7], g = 9.81;
    d[0] = st[3]; d[1] = st[4]; d[2] = st[5];
    d[3] = u[0] * sin(theta) * cos(phi); d[4] = -u[0] * sin(phi);
    d[5] = -g + u[0] * cos(phi) * cos(theta); d[6] = u[1]; d[7] = u[2];
  } else if (ode == OMG_ODE_QUADROTOR2D) {     // quadrotor.py:154-157
    const double theta = st[4], g = 9.81;
    d[0] = st[2]; d[1] = st[3]; d[2] = u[0] * sin(theta); d[3] = u[0] * cos(theta) - g; d[4] = u[1];
  } else if (ode == OMG_ODE_DUBINS) {          // dubins.py: (v cos theta, v sin theta, omega)
    d[0] = u[0] * cos(st[2]); d[1] = u[0] * sin(st[2]); d[2] = u[1];
  } else {                                     // holonomic*.py: state' = input
    for (int j = 0; j < ns; ++j) d[j] = u[j];
  }
}

// Non-ideal prediction: integrate the vehicle ODE over `steps` samples of the planned input
// with classical RK4 (reference Vehicle.predict / integrate_ode, vehicle.py:302-337, 412-423;
// C++ twin Vehicle::integrate, export/vehicles/Vehicle.cpp:80-110: k1..k3 with input[i], k4
// with input[i+1]).  One thread per instance.
__global__ void omg_rk4_kernel(int model, int B, int ns, int ni, const double* __restrict__ state0,
                               const double* __restrict__ inputs, double dt, int steps,
                               double* __restrict__ stateT) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  double x[OMG_ODE_MAX_STATE], k1[OMG_ODE_MAX_STATE], k2[OMG_ODE_MAX_STATE], k3[OMG_ODE_MAX_STATE],
         k4[OMG_ODE_MAX_STATE], st[OMG_ODE_MAX_STATE];
  for (int j = 0; j < ns; ++j) x[j] = state0[(size_t)b * ns + j];
  const double* U = inputs + (size_t)b * (steps + 1) * ni;
  for (int i = 0; i < steps; ++i) {
    const double* u0 = U + (size_t)i * ni;
    const double* u1 = u0 + ni;
    ode_rhs(model, ns, x, u0, k1);
    for (int j = 0; j < ns; ++j) st[j] = x[j] + 0.5 * dt * k1[j];
    ode_rhs(model, ns, st, u0, k2);
    for (int j = 0; j < ns; ++j) st[j] = x[j] + 0.5 * dt * k2[j];
    ode_rhs(model, ns, st, u0, k3);
    for (int j = 0; j < ns; ++j) st[j] = x[j] + dt * k3[j];
    ode_rhs(model, ns, st, u1, k4);
    for (int j = 0; j < ns; ++j) x[j] += (dt / 6.0) * (k1[j] + 2.0 * k2[j] + 2.0 * k3[j] + k4[j]);
  }
  for (int j = 0; j < ns; ++j) stateT[(size_t)b * ns + j] = x[j];
}

// ---- closed-loop plant step (reference Vehicle.simulate / predict without the ideal flags,
// vehicle.py:302-337, 359-449) -----------------------------------------------------------------
#define OMG_CL_MAX_INPUT 3
#define OMG_CL_PAD 12          // filtfilt's odd padding: 3 * max(len(a), len(b)) for butter(3)

// Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC'11): counter
// (sample pair, signal, instance, MPC step), key (seed).  A draw depends on its key and counter
// only, so a realisation is the same at any batch size and under any launch schedule.
__host__ __device__ __forceinline__ void omg_philox4x32_10(uint32_t c[4], uint32_t k0, uint32_t k1) {
  for (int r = 0; r < 10; ++r) {
    if (r) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
    const uint64_t p0 = (uint64_t)0xD2511F53u * c[0], p1 = (uint64_t)0xCD9E8D57u * c[2];
    const uint32_t hi0 = (uint32_t)(p0 >> 32), lo0 = (uint32_t)p0, hi1 = (uint32_t)(p1 >> 32), lo1 = (uint32_t)p1;
    c[0] = hi1 ^ c[1] ^ k0; c[1] = lo1; c[2] = hi0 ^ c[3] ^ k1; c[3] = lo0;
  }
}

// two uniforms in (0, 1) from one Philox block (52 bits each, (m + 1/2) 2^-52, exact), then
// Box-Muller: z0 = r cos(2 pi u2), z1 = r sin(2 pi u2), r = sqrt(-2 log u1)
__device__ __forceinline__ void omg_normal_pair(uint64_t seed, int step, int inst, int sig, int pair,
                                                double* z0, double* z1) {
  uint32_t c[4] = {(uint32_t)pair, (uint32_t)sig, (uint32_t)inst, (uint32_t)step};
  omg_philox4x32_10(c, (uint32_t)seed, (uint32_t)(seed >> 32));
  const double u1 = ((double)(((((uint64_t)c[0] << 32) | c[1]) >> 12)) + 0.5) * 0x1p-52;
  const double u2 = ((double)(((((uint64_t)c[2] << 32) | c[3]) >> 12)) + 0.5) * 0x1p-52;
  const double r = sqrt(-2.0 * log(u1)), w = 6.283185307179586 * u2;
  *z0 = r * cos(w);
  *z1 = r * sin(w);
}

__device__ __forceinline__ double omg_row_dot(const double* r, const double* c, int L) {
  double acc = 0.0;
  for (int k = 0; k < L; ++k) acc += r[k] * c[k];
  return acc;
}

// Planned input of one sample (each vehicle's splines2signals): v[d][c] is the d-th derivative of
// the input spline column c at the sample, divided by T^d.
__device__ __forceinline__ void omg_cl_input_map(int model, int ni, const double (*v)[OMG_CL_MAX_INPUT], double* u) {
  if (model == OMG_ODE_QUADROTOR2D) {               // quadrotor.py splines2signals
    const double ddx = v[2][0], ddy = v[2][1], dddx = v[3][0], dddy = v[3][1];
    const double ay = ddy + 9.81;
    u[0] = sqrt(ddx * ddx + ay * ay);
    u[1] = (dddx * ay - ddx * dddy) / (ay * ay + ddx * ddx);
  } else if (model == OMG_ODE_DUBINS) {             // dubins.py: v = v~ (1 + tg^2), w = 2 tg' / (1 + tg^2)
    const double vt = v[0][0], tg = v[0][1], dtg = v[1][1], q = 1.0 + tg * tg;
    u[0] = vt * q; u[1] = 2.0 * dtg / q;
  } else if (model == OMG_ODE_HOLONOMIC_ORIENT) {   // holonomicorient.py: (x', y', 2 tg' / (1 + tg^2))
    const double tg = v[0][2];
    u[0] = v[1][0]; u[1] = v[1][1];
    u[2] = 2.0 * v[1][2] / (1.0 + tg * tg);
  } else if (model == OMG_ODE_SIMPLE_QUADROTOR3D) { // quadrotor3d_simple.py splines2signals
    const double ddx = v[2][0], ddy = v[2][1], dddx = v[3][0], dddy = v[3][1];
    const double az = v[2][2] + 9.81, dddz = v[3][2];
    const double h2 = ddx * ddx + az * az, f2 = ddx * ddx + ddy * ddy + az * az;
    u[0] = sqrt(f2);
    u[1] = (-dddy * h2 + ddy * (ddx * dddx + dddz * az)) / (f2 * sqrt(h2));
    u[2] = (az * dddx - ddx * dddz) / (az * az + ddx * ddx);
  } else if (model == OMG_ODE_QUADROTOR3D) {
    const double f = v[0][0], qp = v[0][1], qt = v[0][2], dqp = v[1][1], dqt = v[1][2];
    const double ep = 1.0 + qp * qp, et = 1.0 + qt * qt;
    u[0] = f * (ep * et); u[1] = 2.0 * dqp / ep; u[2] = 2.0 * dqt / et;
  } else {
    for (int c = 0; c < ni; ++c) u[c] = v[1][c];
  }
}

// Classical RK4 of the vehicle ODE from the state y over the n_samp sample intervals of the input
// samples U [n_samp+1][ni] on the linearly interpolated input of the reference's interp1d: u_i,
// the mean of u_i and u_i+1 at both midpoints, u_i+1 at the end.  y is updated in place.  The work
// arrays st, k1..k4 [OMG_ODE_MAX_STATE] and um [OMG_CL_MAX_INPUT] are the caller's.
__device__ __forceinline__ void omg_rk4_interp(int ode, int ns, int ni, int n_samp, double dt, const double* U,
                                               double* y, double* st, double* k1, double* k2, double* k3,
                                               double* k4, double* um) {
  for (int i = 0; i < n_samp; ++i) {
    const double* u0 = U + i * ni;
    const double* u1 = u0 + ni;
    for (int c = 0; c < ni; ++c) um[c] = 0.5 * (u0[c] + u1[c]);
    ode_rhs(ode, ns, y, u0, k1);
    for (int j = 0; j < ns; ++j) st[j] = y[j] + 0.5 * dt * k1[j];
    ode_rhs(ode, ns, st, um, k2);
    for (int j = 0; j < ns; ++j) st[j] = y[j] + 0.5 * dt * k2[j];
    ode_rhs(ode, ns, st, um, k3);
    for (int j = 0; j < ns; ++j) st[j] = y[j] + dt * k3[j];
    ode_rhs(ode, ns, st, u1, k4);
    for (int j = 0; j < ns; ++j) y[j] += (dt / 6.0) * (k1[j] + 2.0 * k2[j] + 2.0 * k3[j] + k4[j]);
  }
}

// The part of one instance's plant step that follows the planned inputs U [n_samp+1][ni] (shared
// memory, complete at entry or completed by the caller's threads before the barrier below), run
// by every thread of the block:
//   simulate: planned input + filtered noise -> first-order lag -> RK4 of the ODE -> x_p(t_k+1)
//   predict:  planned input -> RK4 of the ODE from x_p(t_k) -> state0 of the next solve
// RK4 takes the linearly interpolated input of the reference's interp1d: u_i, the mean of
// u_i and u_i+1 at both midpoints, u_i+1 at the end.  The noise series of (instance, signal) is
// filtered over the whole stored trajectory (n_traj samples) by the reference's
// filtfilt(butter(3, fc)): odd extension by 12, forward and backward passes of the transposed
// direct form from zi * (first value); only samples 0..n_samp are kept.
// filt = {b0..b3, a0..a3 (a0 = 1), zi0..zi2}; scratch holds one forward pass per series, `stride`
// doubles apart (at least n_traj + 24).  D, A: [n_samp+1][ni] of shared memory.  p indexes the
// plant arrays ([p][ns], [p][ni]) and the scratch series; the noise of input j is keyed by (seed,
// step, b, sig0 + j, pair), so that the vehicles of a fleet (p = b*n_veh + v, sig0 = v*ni) draw
// their own series and vehicle 0 draws what a single vehicle draws.
__device__ void omg_cl_tail(int b, int p, int sig0, int ode, int ns, int ni, int n_samp, double dt, int lag, double tau,
                            int disturb, int n_traj, const double* __restrict__ filt,
                            const double* __restrict__ mean, const double* __restrict__ stdev, uint64_t seed,
                            int step, const double* plant_x, const double* plant_u, double* plant_x_next,
                            double* plant_u_next, double* __restrict__ pred_x, double* __restrict__ pred_u,
                            double* __restrict__ scratch, size_t stride, const double* U, double* D, double* A) {
  const int ts = n_samp + 1;
  if (disturb && (int)threadIdx.x < ni) {
    const int j = threadIdx.x, N = n_traj + 2 * OMG_CL_PAD;
    double* e = scratch + ((size_t)p * ni + j) * stride;
    double* w = e + OMG_CL_PAD;                     // white noise at 0..n_traj-1
    for (int q = 0; 2 * q < n_traj; ++q) {
      double z0, z1;
      omg_normal_pair(seed, step, b, sig0 + j, q, &z0, &z1);
      w[2 * q] = mean[j] + stdev[j] * z0;
      if (2 * q + 1 < n_traj) w[2 * q + 1] = mean[j] + stdev[j] * z1;
    }
    for (int i = 1; i <= OMG_CL_PAD; ++i) {         // odd extension (scipy odd_ext)
      e[OMG_CL_PAD - i] = 2.0 * w[0] - w[i];
      w[n_traj - 1 + i] = 2.0 * w[n_traj - 1] - w[n_traj - 1 - i];
    }
    const double b0 = filt[0], b1 = filt[1], b2 = filt[2], b3 = filt[3];
    const double a1 = filt[5], a2 = filt[6], a3 = filt[7];
    double z0 = filt[8] * e[0], z1 = filt[9] * e[0], z2 = filt[10] * e[0];
    for (int i = 0; i < N; ++i) {                   // forward pass, in place
      const double xi = e[i], yi = z0 + b0 * xi;
      z0 = z1 + xi * b1 - yi * a1; z1 = z2 + xi * b2 - yi * a2; z2 = xi * b3 - yi * a3;
      e[i] = yi;
    }
    const double y0 = e[N - 1];
    z0 = filt[8] * y0; z1 = filt[9] * y0; z2 = filt[10] * y0;
    for (int i = N - 1; i >= OMG_CL_PAD; --i) {     // backward pass down to sample 0
      const double xi = e[i], yi = z0 + b0 * xi;
      z0 = z1 + xi * b1 - yi * a1; z1 = z2 + xi * b2 - yi * a2; z2 = xi * b3 - yi * a3;
      if (i - OMG_CL_PAD < ts) D[(i - OMG_CL_PAD) * ni + j] = yi;
    }
  }
  double st[OMG_ODE_MAX_STATE], k1[OMG_ODE_MAX_STATE], k2[OMG_ODE_MAX_STATE], k3[OMG_ODE_MAX_STATE],
         k4[OMG_ODE_MAX_STATE], y[OMG_ODE_MAX_STATE], um[OMG_CL_MAX_INPUT];
  // read before the barrier: the outputs may overwrite the plant state in place
  if (threadIdx.x <= 1)
    for (int j = 0; j < ns; ++j) y[j] = plant_x[(size_t)p * ns + j];
  __syncthreads();
  if (threadIdx.x > 1) return;
  const bool simulate = threadIdx.x == 0;
  const double* Uin = U;
  if (simulate) {
    for (int i = 0; i < ts * ni; ++i) A[i] = disturb ? U[i] + D[i] : U[i];
    if (lag) {                                      // u' = (u_cmd - u) / tau from the applied input
      double ua[OMG_CL_MAX_INPUT];
      for (int c = 0; c < ni; ++c) ua[c] = plant_u[(size_t)p * ni + c];
      for (int i = 0; i < n_samp; ++i) {
        for (int c = 0; c < ni; ++c) {
          const double c0 = A[i * ni + c], c1 = A[(i + 1) * ni + c], cm = 0.5 * (c0 + c1), u = ua[c];
          const double q1 = (c0 - u) / tau, q2 = (cm - (u + 0.5 * dt * q1)) / tau;
          const double q3 = (cm - (u + 0.5 * dt * q2)) / tau, q4 = (c1 - (u + dt * q3)) / tau;
          A[i * ni + c] = u;
          ua[c] = u + (dt / 6.0) * (q1 + 2.0 * q2 + 2.0 * q3 + q4);
        }
      }
      for (int c = 0; c < ni; ++c) A[n_samp * ni + c] = ua[c];
    }
    Uin = A;
  }
  omg_rk4_interp(ode, ns, ni, n_samp, dt, Uin, y, st, k1, k2, k3, k4, um);
  double* xo = simulate ? plant_x_next : pred_x;
  double* uo = simulate ? plant_u_next : pred_u;
  for (int j = 0; j < ns; ++j) xo[(size_t)p * ns + j] = y[j];
  for (int c = 0; c < ni; ++c) uo[(size_t)p * ni + c] = Uin[n_samp * ni + c];
}

// One block per (instance b, vehicle v), block p = b*n_veh + v; both halves start from the plant
// state x_p(t_k) and the trajectory just solved, sampled at t_k + s*dt, s = 0..n_samp (omg_cl_tail).
// Vehicle v's input splines are the ni columns of length L at x[b, veh_off[v]...].  R =
// [nd][n_samp+1][L]: row d is the d-th derivative of the basis divided by T^d, nd the rows the
// model reads.  `model` selects the planned-input map, `ode` the right-hand side (omg_ode_models).
// A single vehicle is n_veh = 1 at offset 0.
__global__ void omg_closed_loop_kernel(int model, int ode, int nd, int ns, int ni, int n, int n_veh,
                                       const int* __restrict__ veh_off, const double* __restrict__ x,
                                       int L, int n_samp, const double* __restrict__ R,
                                       double dt, int lag, double tau, int disturb, int n_traj,
                                       const double* __restrict__ filt, const double* __restrict__ mean,
                                       const double* __restrict__ stdev, uint64_t seed, int step,
                                       const double* plant_x, const double* plant_u,    // (may alias the next)
                                       double* plant_x_next, double* plant_u_next,
                                       double* __restrict__ pred_x, double* __restrict__ pred_u,
                                       double* __restrict__ scratch) {
  OMG_DYN_SHARED(sm);
  const int p = blockIdx.x, b = p / n_veh, v = p - b * n_veh, ts = n_samp + 1;
  double* U = sm;                // planned input [ts][ni]
  double* D = sm + ts * ni;      // filtered disturbance [ts][ni]
  double* A = sm + 2 * ts * ni;  // input reaching the ODE [ts][ni]
  const double* xb = x + (size_t)b * n + veh_off[v];
  const size_t nr = (size_t)ts * L;
  for (int s = threadIdx.x; s < ts; s += blockDim.x) {
    double v[4][OMG_CL_MAX_INPUT];
    for (int d = 0; d < nd; ++d)
      for (int c = 0; c < ni; ++c) v[d][c] = omg_row_dot(R + d * nr + (size_t)s * L, xb + c * L, L);
    omg_cl_input_map(model, ni, v, U + s * ni);
  }
  omg_cl_tail(b, p, v * ni, ode, ns, ni, n_samp, dt, lag, tau, disturb, n_traj, filt, mean, stdev, seed, step,
              plant_x, plant_u, plant_x_next, plant_u_next, pred_x, pred_u, scratch, (size_t)n_traj + 2 * OMG_CL_PAD,
              U, D, A);
}

// trajectory sampling: out[b, blk, c, s] = sum_k S_blk[s,k] * x[b, off_blk + c*len_blk + k]
// (batched Cox-de Boor evaluation with precomputed basis rows; reference
//  Vehicle.store -> sample_splines, vehicle.py:250-300, spline_extra.py:406-410;
//  C++ twin Vehicle::sampleSplines, Vehicle.cpp:112-190)
__global__ void omg_sample_kernel(const double* __restrict__ x, int B, int n, int n_blocks,
                                  const int* __restrict__ offs, const int* __restrict__ lens,
                                  const int* __restrict__ ncols, const int* __restrict__ nsamp,
                                  const int* __restrict__ soffs, const int* __restrict__ ooffs,
                                  const double* __restrict__ Sm, double* __restrict__ out, int n_out) {
  OMG_DYN_SHARED(xs);
  const int b = blockIdx.x;
  if (b >= B) return;
  const double* xb = x + (size_t)b * n;
  for (int i = threadIdx.x; i < n; i += blockDim.x) xs[i] = xb[i];
  __syncthreads();
  double* ob = out + (size_t)b * n_out;
  for (int blk = 0; blk < n_blocks; ++blk) {
    const int L = lens[blk], nc = ncols[blk], ns = nsamp[blk], off = offs[blk];
    const double* Sb = Sm + soffs[blk];
    for (int e = threadIdx.x; e < ns * nc; e += blockDim.x) {
      const int c = e / ns, sidx = e - c * ns;
      double acc = 0.0;
      for (int k = 0; k < L; ++k) acc += Sb[sidx * L + k] * xs[off + c * L + k];
      ob[ooffs[blk] + c * ns + sidx] = acc;
    }
  }
}

// ---------------------------------------------------------------------------
// Per-instance spline bases (free motion time: every instance has its own tau = dt / T_b, so no
// basis row can be shared across the batch).  Block descriptors are 6 ints per spline variable:
// {offset in x, basis length L, columns, degree p, offset of its L + p + 1 knots, offset of its
// derivative coefficients in shared memory (omg_eval_kernel)}.
// ---------------------------------------------------------------------------
#ifdef OMG_CPU_EMU
static inline double __dadd_rn(double a, double b) { return a + b; }   // (__dmul_rn: omg_sp.cuh)
#endif
#define OMG_SPL_DESC 6
#define OMG_SPL_GRID 501      // NO_POINTS of basics/spline.py: the collocation grid
#define OMG_SPL_DROP 1e-10    // _DROP_TOL of basics/spline.py

// Cox-de Boor recursion of BSplineBasis.eval_basis (basics/spline.py; reference spline.py:131-136,
// 214-233) for the basis functions i0 .. i0+cnt-1 of degree p on the knots k: w holds cnt + p
// doubles, the values end in w[0..cnt).  The leading clamped intervals (i < p + 1 and k[i] == k[0])
// are closed on both ends, every other interval is (k_i, k_i+1]; zero-length spans are skipped
// (den == 0).  Each value is rounded in the order numpy rounds it (no contraction into an FMA), so
// the values are the host's bit for bit: the collocation points of omg_shift_free_kernel are
// arg-max positions and depend on ties between them.
__device__ void omg_cox_de_boor(const double* k, int p, double x, int i0, int cnt, double* w) {
  for (int j = 0; j < cnt + p; ++j) {
    const int i = i0 + j;
    const bool closed = i < p + 1 && k[0] == k[i];
    w[j] = ((closed ? x >= k[i] : x > k[i]) && x <= k[i + 1]) ? 1.0 : 0.0;
  }
  for (int d = 1; d <= p; ++d)
    for (int j = 0; j < cnt + p - d; ++j) {      // (w[j + 1] is still the previous degree's)
      const int i = i0 + j;
      double acc = 0.0, den = k[i + d] - k[i];
      if (den != 0.0) acc = __dadd_rn(acc, __dmul_rn(x - k[i], w[j]) / den);
      den = k[i + d + 1] - k[i + 1];
      if (den != 0.0) acc = __dadd_rn(acc, __dmul_rn(k[i + d + 1] - x, w[j + 1]) / den);
      w[j] = acc;
    }
}

// numpy.linspace(a, b, num)[i]: i * ((b - a) / (num - 1)) + a, and b itself at the end
__device__ __forceinline__ double omg_linspace(double a, double b, int num, int i) {
  return i == num - 1 ? b : __dadd_rn(__dmul_rn((double)i, (b - a) / (double)(num - 1)), a);
}

// The update u and target time of a free-T warm start from the motion time T (reference
// FreeTPoint2point.init_step, point2point.py:354-368): u = T - dt, target = T when T < 2 dt; else
// u = dt, target = T - dt.  Returns tau = u / target.
__device__ __forceinline__ double omg_free_shift_tau(double T, double dt, double* target) {
  double u = dt;
  *target = T - dt;
  if (T < 2.0 * dt) { u = T - dt; *target = T; }
  return u / *target;
}

// Free-T re-expression of one x row by the threads of a block (shift_spline, spline_extra.py:88-99):
// every block is re-expressed on shift_spline's basis
//   knots2 = [tau] * p + linspace(tau, end, L - p + 1) + [end] * p
// by BSplineBasis.transform: collocation at the first arg-max of each new basis function over
// linspace(tau, end, 501), M = bm^-1 old_basis(points), entries below 1e-10 dropped, c <- M c.
// xs: the source row in shared memory, loaded by the caller (the first barrier below orders it);
// xb: the destination row (must not alias xs).  sm: shared scratch of knots2 [Lmax + pmax + 1] |
// points [Lmax] | arg-max scratch [2 blockDim] | bm [Lmax^2] | old_basis(points), then M [Lmax^2].
__device__ __forceinline__ void omg_shift_free_row(const double* xs, double* xb, double tau, int n_blocks,
                                                   const int* __restrict__ desc, const double* __restrict__ kn,
                                                   int Lmax, int pmax, double* sm) {
  const int t = threadIdx.x, nt = blockDim.x;
  double* k2 = sm;
  double* xm = k2 + Lmax + pmax + 1;
  double* sv = xm + Lmax;
  double* sg = sv + nt;
  double* A = sg + nt;
  double* R = A + (size_t)Lmax * Lmax;
  for (int blk = 0; blk < n_blocks; ++blk) {
    const int* dsc = desc + OMG_SPL_DESC * blk;
    const int off = dsc[0], L = dsc[1], nc = dsc[2], p = dsc[3];
    const double* ko = kn + dsc[4];
    const double end = ko[L + p];
    const int nk = L - p + 1;
    __syncthreads();                              // (x row loaded / previous block done)
    for (int j = t; j < L + p + 1; j += nt)
      k2[j] = j < p ? tau : (j < p + nk ? omg_linspace(tau, end, nk, j - p) : end);
    __syncthreads();
    // collocation points: S segments of the grid per basis function, the first maximum of each
    // segment, then the first maximum over the segments in grid order (numpy.argmax)
    const int S = nt / L > 0 ? nt / L : 1, seg = (OMG_SPL_GRID + S - 1) / S;
    if (t < L * S) {
      const int l = t % L, s = t / L;
      double w[OMG_SPL_MAX_DEGREE + 1], best = -1.0;
      int bg = -1;
      const int g1 = min(OMG_SPL_GRID, (s + 1) * seg);
      for (int g = s * seg; g < g1; ++g) {
        const double xg = omg_linspace(tau, end, OMG_SPL_GRID, g);
        double v = 0.0;                           // (exactly 0 outside the support)
        if (xg >= k2[l] && xg <= k2[l + p + 1]) { omg_cox_de_boor(k2, p, xg, l, 1, w); v = w[0]; }
        if (v > best) { best = v; bg = g; }
      }
      sv[t] = best; sg[t] = (double)bg;
    }
    __syncthreads();
    for (int l = t; l < L; l += nt) {
      double best = -1.0; int bg = 0;
      for (int s = 0; s < S; ++s)
        if (sg[s * L + l] >= 0.0 && sv[s * L + l] > best) { best = sv[s * L + l]; bg = (int)sg[s * L + l]; }
      xm[l] = omg_linspace(tau, end, OMG_SPL_GRID, bg);
    }
    __syncthreads();
    // bm = new_basis(points), R = old_basis(points)
    for (int i = t; i < L; i += nt) {
      double w[OMG_SPL_MAX_LEN + OMG_SPL_MAX_DEGREE];
      omg_cox_de_boor(k2, p, xm[i], 0, L, w);
      for (int l = 0; l < L; ++l) A[i * L + l] = w[l];
      omg_cox_de_boor(ko, p, xm[i], 0, L, w);
      for (int l = 0; l < L; ++l) R[i * L + l] = w[l];
    }
    // bm M = R by Gaussian elimination WITHOUT pivoting: a collocation matrix of a B-spline basis
    // at points that satisfy Schoenberg-Whitney (each point inside its function's support) is
    // banded and totally positive, and for such matrices elimination without pivoting is stable
    // (de Boor & Pinkus 1977).  The host's LU with partial pivoting rounds differently.
    for (int j = 0; j < L - 1; ++j) {
      __syncthreads();
      const double piv = A[j * L + j];
      const int nr = L - 1 - j, wa = L - 1 - j, wr = wa + L;
      for (int e = t; e < nr * wr; e += nt) {
        const int i = j + 1 + e / wr, c = e % wr;
        const double f = A[i * L + j] / piv;
        if (c < wa) A[i * L + j + 1 + c] -= f * A[j * L + j + 1 + c];
        else R[i * L + c - wa] -= f * R[j * L + c - wa];
      }
    }
    __syncthreads();
    for (int c = t; c < L; c += nt)
      for (int i = L - 1; i >= 0; --i) {
        double s = R[i * L + c];
        for (int k = i + 1; k < L; ++k) s -= A[i * L + k] * R[k * L + c];
        R[i * L + c] = s / A[i * L + i];
      }
    __syncthreads();
    for (int e = t; e < L * nc; e += nt) {
      const int c = e / L, i = e - c * L;
      double acc = 0.0;
      for (int k = 0; k < L; ++k) {
        const double m = R[i * L + k];
        if (fabs(m) >= OMG_SPL_DROP) acc += m * xs[off + c * L + k];
      }
      xb[off + c * L + i] = acc;
    }
  }
}

// Free-T warm start of one instance per block (reference FreeTPoint2point.init_step with
// shift_spline): tau from T = x[t_index] (omg_free_shift_tau), the row re-expressed in place
// (omg_shift_free_row), then x[t_index] = target.  Inactive instances and tau outside (0, 1) are
// left alone.  Shared memory: x row [n] | the scratch of omg_shift_free_row.
__global__ void omg_shift_free_kernel(double* x, int B, int n, int t_index, double dt,
                                      const int* __restrict__ active, int n_blocks,
                                      const int* __restrict__ desc, const double* __restrict__ kn,
                                      int Lmax, int pmax) {
  OMG_DYN_SHARED(xs);
  const int b = blockIdx.x, t = threadIdx.x, nt = blockDim.x;
  if (b >= B || (active && !active[b])) return;
  double* xb = x + (size_t)b * n;
  double target;
  const double tau = omg_free_shift_tau(xb[t_index], dt, &target);
  if (!(tau > 0.0 && tau < 1.0)) return;
  for (int i = t; i < n; i += nt) xs[i] = xb[i];
  omg_shift_free_row(xs, xb, tau, n_blocks, desc, kn, Lmax, pmax, xs + n);
  __syncthreads();                                // (every thread has read T)
  if (t == 0) xb[t_index] = target;
}

// Derivative coefficients of one spline column c [L] of degree p on the knots k, the arithmetic of
// omg_eval_kernel and omg_closed_loop_free_kernel (which keep their own inline copies: routed through
// this function, their generated code changes): row d of q [n_der][L] holds the L - d coefficients
// of the d-th derivative.
__device__ __forceinline__ void omg_spl_der_coef(const double* k, int p, int L, int n_der, const double* c, double* q) {
  for (int i = 0; i < L; ++i) q[i] = c[i];
  for (int d = 1; d < n_der; ++d)
    for (int j = 0; j < L - d; ++j) {
      const double den = k[j + p + 1] - k[j + d];
      q[d * L + j] = den != 0.0 ? (p - d + 1) * (q[(d - 1) * L + j + 1] - q[(d - 1) * L + j]) / den : 0.0;
    }
}

// Per-instance evaluation, one instance per block: out[b, blk, c, j, d] = d-th derivative of
// column c of block blk at tau[b, j], divided by scale[b]^d (d < n_der).  Derivatives as
// BSplineBasis.derivative takes them (de Boor X.16): coefficients c' = (p - i) (c_j+1 - c_j) /
// (k_j+p+1 - k_j+i+1) per order i on the basis of degree p - d and knots k[d : -d]; a span of
// zero length gives a zero coefficient (its basis function vanishes).
__global__ void omg_eval_kernel(const double* __restrict__ x, int B, int n, int n_blocks,
                                const int* __restrict__ desc, const double* __restrict__ kn, int n_pts,
                                const double* __restrict__ tau, const double* __restrict__ scale,
                                int n_der, double* __restrict__ out, int n_out) {
  OMG_DYN_SHARED(cd);                       // per block and column: n_der rows of L coefficients
  const int b = blockIdx.x, t = threadIdx.x, nt = blockDim.x;
  if (b >= B) return;
  const double* xb = x + (size_t)b * n;
  int n_col = 0;
  for (int blk = 0; blk < n_blocks; ++blk) n_col += desc[OMG_SPL_DESC * blk + 2];
  for (int e = t; e < n_col; e += nt) {
    int blk = 0, c = e;
    while (c >= desc[OMG_SPL_DESC * blk + 2]) c -= desc[OMG_SPL_DESC * blk++ + 2];
    const int* dsc = desc + OMG_SPL_DESC * blk;
    const int L = dsc[1], p = dsc[3];
    const double* k = kn + dsc[4];
    double* q = cd + dsc[5] + (size_t)c * n_der * L;
    for (int i = 0; i < L; ++i) q[i] = xb[dsc[0] + c * L + i];
    for (int d = 1; d < n_der; ++d)
      for (int j = 0; j < L - d; ++j) {
        const double den = k[j + p + 1] - k[j + d];
        q[d * L + j] = den != 0.0 ? (p - d + 1) * (q[(d - 1) * L + j + 1] - q[(d - 1) * L + j]) / den : 0.0;
      }
  }
  __syncthreads();
  const double s = scale[b];
  double* ob = out + (size_t)b * n_out;
  int ooff = 0;
  for (int blk = 0; blk < n_blocks; ++blk) {
    const int* dsc = desc + OMG_SPL_DESC * blk;
    const int L = dsc[1], nc = dsc[2], p = dsc[3];
    const double* k = kn + dsc[4];
    for (int j = t; j < n_pts; j += nt) {
      const double xj = tau[(size_t)b * n_pts + j];
      double w[OMG_SPL_MAX_LEN + OMG_SPL_MAX_DEGREE], sd = 1.0;
      for (int d = 0; d < n_der; ++d) {
        omg_cox_de_boor(k + d, p - d, xj, 0, L - d, w);
        for (int c = 0; c < nc; ++c) {
          const double* q = cd + dsc[5] + ((size_t)c * n_der + d) * L;
          double acc = 0.0;
          for (int i = 0; i < L - d; ++i) acc += w[i] * q[i];
          ob[ooff + ((size_t)c * n_pts + j) * n_der + d] = acc / sd;
        }
        sd *= s;
      }
    }
    ooff += nc * n_pts * n_der;
  }
}

// Closed-loop plant step with a free motion time, one instance per block: omg_closed_loop_kernel
// with the planned inputs of instance b sampled on its own time axis, s*dt / T_b for
// s = 0..n_samp[b], T_b = x[b, t_index], by the derivative coefficients and Cox-de Boor values of
// omg_eval_kernel (derivative d divided by T_b^d).  desc = {offset in x, L, columns, degree} of the
// spline block whose first ni columns are the input splines, kn its L + p + 1 knots.  n_samp[b] = 0:
// nothing is written for b; n_traj[b] = 0: no disturbance for b.  Shared memory: U, D, A
// [ts_max][ni] | derivative coefficients [ni][nd][L].
__global__ void omg_closed_loop_free_kernel(int model, int ode, int nd, int ns, int ni, int n,
                                            const double* __restrict__ x, const int* __restrict__ desc,
                                            const double* __restrict__ kn, int t_index,
                                            const int* __restrict__ n_samp, const int* __restrict__ n_traj,
                                            int ts_max, double dt, int lag, double tau, int disturb,
                                            const double* __restrict__ filt, const double* __restrict__ mean,
                                            const double* __restrict__ stdev, uint64_t seed, int step,
                                            const double* plant_x, const double* plant_u,
                                            double* plant_x_next, double* plant_u_next,
                                            double* __restrict__ pred_x, double* __restrict__ pred_u,
                                            double* __restrict__ scratch, size_t stride) {
  OMG_DYN_SHARED(sm);
  const int b = blockIdx.x, t = threadIdx.x, nt = blockDim.x, nsb = n_samp[b];
  if (nsb <= 0) return;
  const int ts = nsb + 1, off = desc[0], L = desc[1], p = desc[3];
  double* U = sm;
  double* D = sm + (size_t)ts_max * ni;
  double* A = sm + 2 * (size_t)ts_max * ni;
  double* cd = sm + 3 * (size_t)ts_max * ni;
  const double* xb = x + (size_t)b * n;
  const double T = xb[t_index];
  for (int c = t; c < ni; c += nt) {                // de Boor X.16, as omg_eval_kernel
    double* q = cd + (size_t)c * nd * L;
    for (int i = 0; i < L; ++i) q[i] = xb[off + c * L + i];
    for (int d = 1; d < nd; ++d)
      for (int j = 0; j < L - d; ++j) {
        const double den = kn[j + p + 1] - kn[j + d];
        q[d * L + j] = den != 0.0 ? (p - d + 1) * (q[(d - 1) * L + j + 1] - q[(d - 1) * L + j]) / den : 0.0;
      }
  }
  __syncthreads();
  for (int s = t; s < ts; s += nt) {
    const double xs = (double)s * dt / T;
    double w[OMG_SPL_MAX_LEN + OMG_SPL_MAX_DEGREE], v[4][OMG_CL_MAX_INPUT], sd = 1.0;
    for (int d = 0; d < nd; ++d) {
      omg_cox_de_boor(kn + d, p - d, xs, 0, L - d, w);
      for (int c = 0; c < ni; ++c) {
        const double* q = cd + ((size_t)c * nd + d) * L;
        double acc = 0.0;
        for (int i = 0; i < L - d; ++i) acc += w[i] * q[i];
        v[d][c] = acc / sd;
      }
      sd *= T;
    }
    omg_cl_input_map(model, ni, v, U + s * ni);
  }
  const int ntr = n_traj ? n_traj[b] : 0;
  omg_cl_tail(b, b, 0, ode, ns, ni, nsb, dt, lag, tau, disturb && ntr > 0, ntr, filt, mean, stdev, seed, step, plant_x,
              plant_u, plant_x_next, plant_u_next, pred_x, pred_u, scratch, stride, U, D, A);
}

// ---------------------------------------------------------------------------
// ADMM consensus step of one agent per block (reference admm.py:117-168 z-update,
// 248-266 lambda-update, 268-307 residuals), in first-knot-shifted coordinates:
//   v   = Tf (x + l/rho)            for the own copy and every neighbour copy
//   z~  = P v + c                   P = I - A^T (A A^T)^-1 A,  c = A^T (A A^T)^-1 b
//   z   = Tb z~ ;  l += rho (x - z)
//   pr  = |Tf (x - z)|^2 ; dr = rho |Tf (z - z_prev)|^2 ; cr = rho pr + dr
// Tf / Tb (L x L, row-major) restrict a spline to the future / undo it.
// ---------------------------------------------------------------------------
__global__ void omg_admm_zl_kernel(int nsh, int nn, int L, const double* __restrict__ PzT,
                                   const double* __restrict__ c, const double* __restrict__ Tf,
                                   const double* __restrict__ Tb, double rho,
                                   const double* __restrict__ x_i, const double* __restrict__ x_j,
                                   double* __restrict__ z_i, double* __restrict__ z_ij,
                                   double* __restrict__ l_i, double* __restrict__ l_ij,
                                   double* __restrict__ res) {
  OMG_DYN_SHARED(sh);
  const int nz = nsh * (1 + nn);
  double* xs = sh;            // x  (own, neighbours)      [nz]
  double* ls = xs + nz;       // l                          [nz]
  double* zp = ls + nz;       // previous z                 [nz]
  double* v = zp + nz;        // Tf (x + l/rho)             [nz]
  double* zt = v + nz;        // z~ then z                  [nz]
  double* red = zt + nz;      // [2 * blockDim/32]
  const int a = blockIdx.x, tid = threadIdx.x;
  for (int k = tid; k < nz; k += blockDim.x) {
    const bool own = k < nsh;
    xs[k] = own ? x_i[(size_t)a * nsh + k] : x_j[(size_t)a * nn * nsh + (k - nsh)];
    ls[k] = own ? l_i[(size_t)a * nsh + k] : l_ij[(size_t)a * nn * nsh + (k - nsh)];
    zp[k] = own ? z_i[(size_t)a * nsh + k] : z_ij[(size_t)a * nn * nsh + (k - nsh)];
  }
  __syncthreads();
  for (int k = tid; k < nz; k += blockDim.x) {       // v = Tf (x + l/rho), spline by spline
    const int blk = k / L, r = k - blk * L;
    double acc = 0.0;
    for (int q = 0; q < L; ++q) acc += Tf[r * L + q] * (xs[blk * L + q] + ls[blk * L + q] / rho);
    v[k] = acc;
  }
  __syncthreads();
  for (int k = tid; k < nz; k += blockDim.x) {       // z~ = P v + c
    double acc = c[(size_t)a * nz + k];
    for (int q = 0; q < nz; ++q) acc += PzT[(size_t)q * nz + k] * v[q];
    zt[k] = acc;
  }
  __syncthreads();
  double znew = 0.0;
  for (int k = tid; k < nz; k += blockDim.x) {       // z = Tb z~ (one entry per thread, nz <= blockDim)
    const int blk = k / L, r = k - blk * L;
    double acc = 0.0;
    for (int q = 0; q < L; ++q) acc += Tb[r * L + q] * zt[blk * L + q];
    znew = acc;
  }
  __syncthreads();
  for (int k = tid; k < nz; k += blockDim.x) zt[k] = znew;
  __syncthreads();
  double pr = 0.0, dr = 0.0;
  for (int k = tid; k < nz; k += blockDim.x) {
    const bool own = k < nsh;
    const double zk = zt[k];
    const double lk = ls[k] + rho * (xs[k] - zk);
    if (own) { z_i[(size_t)a * nsh + k] = zk; l_i[(size_t)a * nsh + k] = lk; }
    else { z_ij[(size_t)a * nn * nsh + (k - nsh)] = zk; l_ij[(size_t)a * nn * nsh + (k - nsh)] = lk; }
    const int blk = k / L, r = k - blk * L;
    double e1 = 0.0, e2 = 0.0;
    for (int q = 0; q < L; ++q) {
      const double t = Tf[r * L + q];
      e1 += t * (xs[blk * L + q] - zt[blk * L + q]);
      e2 += t * (zt[blk * L + q] - zp[blk * L + q]);
    }
    pr += e1 * e1; dr += rho * e2 * e2;
  }
  for (int off = 16; off > 0; off >>= 1) { pr += __shfl_down_sync(FULL, pr, off); dr += __shfl_down_sync(FULL, dr, off); }
  const int nw = blockDim.x >> 5;
  if ((tid & 31) == 0) { red[tid >> 5] = pr; red[nw + (tid >> 5)] = dr; }
  __syncthreads();
  if (tid == 0) {
    double p = 0.0, d = 0.0;
    for (int w = 0; w < nw; ++w) { p += red[w]; d += red[nw + w]; }
    res[(size_t)a * 3 + 0] = p; res[(size_t)a * 3 + 1] = d; res[(size_t)a * 3 + 2] = rho * p + d;
  }
}

// ---------------------------------------------------------------------------
// Feasibility phase (fallback after Restoration_Failed; oracle/ipm_ref.py feasibility_lm):
// Levenberg-Marquardt on the constraint violation v(x) = g - clip(g, lbg, ubg),
//   (Jv^T Jv + lam I) dx = -Jv^T v,   Jv = the rows with v != 0,
// accept x + dx when it lowers 1/2 |v|^2 (then lam /= 10), else lam *= 10 (12 tries).
// One block per instance at a time; everything lives in the block's L2-resident scratch:
//   V[n_v] | jx[nnz_jx] | v[m] | vt[m] | A[n*n] | L[(n+1)*n] | rhs[n] | dx[n] | xe[n_xe] | xt[n_xe]
// A is assembled one thread per column through the CSC view of the Jacobian (no atomics:
// the sums are in a fixed order), the dense Cholesky carries the right-hand side as row n.
// ---------------------------------------------------------------------------
struct FeasArgs {
  int B, bounds_shared, max_steps;
  const double *x0, *p, *lbg, *ubg;
  double *x, *viol; int* steps;
  double* scr; size_t stride;
};

__device__ __forceinline__ double feas_viol(double g, double lb, double ub) {
  return (g < lb) ? g - lb : ((g > ub) ? g - ub : 0.0);
}

// v[i] for the point xq (mids of xq refreshed first); returns 1/2 |v|^2 and max |v| to all threads
__device__ __forceinline__ void feas_residual(const DevTab& T, const double* V, double* xq, const double* lbg,
                                              const double* ubg, double* v, double* red, double* phi, double* vmax) {
  const int tid = threadIdx.x;
  for (int l = tid; l < T.n_mid; l += NT) { const int2 r = T.midg[l]; xq[T.n + 1 + l] = eval_range(T.Gt, r.x, r.y, V, xq); }
  __syncthreads();
  double ss = 0.0, mx = 0.0;
  for (int i = tid; i < T.m; i += NT) {
    const RowRec rr = T.rowrec[i];
    const double vi = feas_viol(eval_range(T.Gt, rr.g0, rr.g1, V, xq), lbg[i], ubg[i]);
    v[i] = vi; ss += vi * vi; mx = fmax(mx, fabs(vi));
  }
  double r2[2] = {ss, mx};
  block_reduce<OP_SUM, OP_MAX>(r2, red);
  *phi = 0.5 * r2[0]; *vmax = r2[1];
}

__global__ void __launch_bounds__(256, 2)
omg_feas_kernel(const DevTab T, const FeasArgs F) {
  __shared__ double red[MAX_NWARP * 2];
  __shared__ double piv_s;
  const int tid = threadIdx.x;
  const int n = T.n, m = T.m, n_xe = T.n + 1 + T.n_mid;
  double* D = F.scr + (size_t)blockIdx.x * F.stride;
  double* V = D;            double* jx = V + T.n_v;     double* v = jx + T.nnz_jx;
  double* vt = v + m;       double* Am = vt + m;        double* L = Am + (size_t)n * n;
  double* rhs = L + (size_t)(n + 1) * n;  double* dx = rhs + n;
  double* xe = dx + n;      double* xt = xe + n_xe;
  for (int inst = blockIdx.x; inst < F.B; inst += gridDim.x) {
    const double* par = F.p + (size_t)inst * T.n_par;
    const double* lbg = F.lbg + (F.bounds_shared ? 0 : (size_t)inst * m);
    const double* ubg = F.ubg + (F.bounds_shared ? 0 : (size_t)inst * m);
    for (int i = tid; i < 1 + T.n_par; i += NT) V[i] = (i == 0) ? 1.0 : par[i - 1];
    __syncthreads();
    for (int l = 0; l < T.n_levels; ++l) {      // parameter tape (as ipm_body S1)
      for (int e = T.level_ptr[l] + tid; e < T.level_ptr[l + 1]; e += NT) {
        double acc = 0.0;
        for (int t = T.tape_ptr[e]; t < T.tape_ptr[e + 1]; ++t) {
          const int4 f = __ldg(reinterpret_cast<const int4*>(T.tape_fac) + t);
          acc += T.tape_coef[t] * V[f.x] * V[f.y] * V[f.z] * V[f.w];
        }
        switch (T.tape_func[e]) {
          case 1: acc = 1.0 / acc; break;
          case 2: acc = (acc >= 0.0) ? 1.0 : 0.0; break;
          case 3: acc = (acc > 0.0) ? 1.0 : 0.0; break;
          case 4: acc = sin(acc); break;
          case 5: acc = cos(acc); break;
          case 6: acc = sqrt(acc); break;
          default: break;
        }
        V[1 + T.n_par + e] = acc;
      }
      __syncthreads();
    }
    for (int i = tid; i < n_xe; i += NT) {
      const double xi = (i < n) ? F.x0[(size_t)inst * n + i] : ((i == n) ? 1.0 : 0.0);
      xe[i] = xi; xt[i] = xi;
    }
    __syncthreads();
    double phi, vmax, lam = 1e-3;
    feas_residual(T, V, xe, lbg, ubg, v, red, &phi, &vmax);
    int steps = 0;
    while (steps < F.max_steps && vmax > 1e-8) {
      jac_xl(T, V, xe, jx, jx, nullptr, true);           // jx[0..nnz_j) = Jacobian slots (jval aliases jx)
      // normal equations, thread c owns row c of A: sum over the active rows of column c
      for (int c = tid; c < n; c += NT) {
        double* Ac = Am + (size_t)c * n;
        for (int k = 0; k < n; ++k) Ac[k] = 0.0;
        double bc = 0.0;
        for (int q = T.colptr[c]; q < T.colptr[c + 1]; ++q) {
          const unsigned cr = __ldg(T.colrec + q);
          const int s1 = (int)(cr & 0xffffu), r = (int)(cr >> 16);
          const double vr = v[r];
          if (vr == 0.0) continue;
          const double j1 = jx[s1];
          bc -= j1 * vr;
          const RowRec rr = T.rowrec[r];
          for (int k = 0; k < rr.ns; ++k) Ac[T.jcol16[rr.s0 + k]] += j1 * jx[rr.s0 + k];
        }
        rhs[c] = bc;
      }
      __syncthreads();
      bool accepted = false;
      for (int attempt = 0; attempt < 12 && !accepted; ++attempt) {
        // L = lower(A) + lam I, row n = rhs
        for (int e = tid; e < (n + 1) * n; e += NT) {
          const int i = e / n, k = e - i * n;
          L[e] = (i == n) ? rhs[k] : ((k <= i) ? Am[e] + ((k == i) ? lam : 0.0) : 0.0);
        }
        __syncthreads();
        bool ok = true;
        for (int j = 0; j < n; ++j) {
          if (tid == 0) {
            const double d = L[(size_t)j * n + j];
            const double pv = (d > 0.0 && d < 1e300) ? sqrt(d) : -1.0;
            piv_s = pv;
            if (pv > 0.0) L[(size_t)j * n + j] = pv;
          }
          __syncthreads();
          const double pv = piv_s;
          if (!(pv > 0.0)) { ok = false; break; }
          const double inv = 1.0 / pv;
          for (int i = j + 1 + tid; i <= n; i += NT) L[(size_t)i * n + j] *= inv;
          __syncthreads();
          for (int i = j + 1 + tid; i <= n; i += NT) {
            double* Li = L + (size_t)i * n;
            const double lij = Li[j];
            const int kend = (i < n) ? i : n - 1;
            for (int k = j + 1; k <= kend; ++k) Li[k] -= lij * L[(size_t)k * n + j];
          }
          __syncthreads();
        }
        __syncthreads();
        double pt = 0.0, vmt = 0.0;
        if (ok) {
          // back substitution L^T dx = w (w = row n)
          double* w = L + (size_t)n * n;
          for (int j = n - 1; j >= 0; --j) {
            if (tid == 0) dx[j] = w[j] / L[(size_t)j * n + j];
            __syncthreads();
            const double dj = dx[j];
            for (int k = tid; k < j; k += NT) w[k] -= L[(size_t)j * n + k] * dj;
            __syncthreads();
          }
          for (int i = tid; i < n; i += NT) xt[i] = xe[i] + dx[i];
          __syncthreads();
          feas_residual(T, V, xt, lbg, ubg, vt, red, &pt, &vmt);
        }
        if (ok && pt < phi) {          // (a NaN pt compares false)
          for (int i = tid; i < n_xe; i += NT) xe[i] = xt[i];
          for (int i = tid; i < m; i += NT) v[i] = vt[i];
          phi = pt; vmax = vmt; lam = fmax(lam / 10.0, 1e-12);
          accepted = true;
        } else {
          lam *= 10.0;
        }
        __syncthreads();
      }
      if (!accepted) break;
      ++steps;
    }
    for (int i = tid; i < n; i += NT) F.x[(size_t)inst * n + i] = xe[i];
    if (tid == 0) { F.viol[inst] = vmax; F.steps[inst] = steps; }
    __syncthreads();
  }
}


// ===========================================================================
// host side: C ABI
// ===========================================================================
static thread_local std::string g_err;
static void set_err(const std::string& s) { g_err = s; }
#define CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { \
  set_err(std::string(#call) + ": " + cudaGetErrorString(e_)); return -1; } } while (0)

// Device buffers for the block descriptors of the shift / sampling calls.  They only GROW (a
// receding-horizon loop passes the same block layout every step, the sampling matrix changes
// with the time): after the first call there is no cudaMalloc / cudaFree, and the small
// host-to-device copies are enqueued on the CALLER's stream every time, so calls on different
// streams are ordered correctly and stay asynchronous.
struct DescCache {
  int device = -1;
  size_t cap_i = 0, cap_d = 0;
  int* d_i = nullptr; double* d_d = nullptr;
  ~DescCache() { if (d_i) cudaFree(d_i); if (d_d) cudaFree(d_d); }
};

static void free_desc(DescCache* c) { delete c; }

struct omg_problem {
  int device = 0;
  DevTab T;
  Smem S;
  omg_options opt;
  std::vector<void*> allocs;
  int n_sm = 0, ctas_per_sm = 1, nt = 512, target_ctas = 1;
  bool xl = false;
  size_t smem_bytes = 0;
  double* dscr = nullptr; int* iscr = nullptr; int scr_ctas = 0;
  int dscr_stride = 0, iscr_stride = 0;
  int* counter = nullptr; double* trace = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  bool timed = false; int launches = 0;
  // staging buffers for the _host entry point
  double *hx0 = nullptr, *hp = nullptr, *hlb = nullptr, *hub = nullptr, *hlam0 = nullptr,
         *hx = nullptr, *hlam = nullptr, *hf = nullptr;
  int *hst = nullptr, *hit = nullptr; int hostB = 0, host_shared = -1;
  // scratch of the feasibility phase (omg_feas_batch), sized on first use
  double* fscr = nullptr; int fscr_ctas = 0; size_t fscr_stride = 0;
  DescCache* shift_desc = nullptr;   // device copy of the last omg_shift_batch block descriptor
  const double* lbg = nullptr; const double* ubg = nullptr;   // the tables' bounds (omg_mpc_update)
  // sparse kernel variant (omg_sp.cuh / omg_sp_host.cuh)
  bool sp = false; SpTab P; SpSmem SS; size_t sp_smem_bytes = 0; int sp_ctas = 0, sp_dscr_stride = 0;
  std::string sp_info, sp_info_extra;
  // launch configuration of the envelope kernels (kept: inertia_mode = 1 is tied to the
  // envelope's elimination order and always runs there)
  int env_nt = 0, env_ctas = 0; size_t env_smem_bytes = 0;
  bool wide = false;   // factor_env's strided panel solve (WIDE instantiation of the envelope kernels)
  std::string env_info;   // omg_envelope_layout
};

template <typename Tp>
static const Tp* upload(omg_problem* h, const Tp* src, size_t count, bool* ok) {
  if (count == 0) count = 1;
  void* d = nullptr;
  if (cudaMalloc(&d, count * sizeof(Tp)) != cudaSuccess) { *ok = false; return nullptr; }
  h->allocs.push_back(d);
  if (src && cudaMemcpy(d, src, count * sizeof(Tp), cudaMemcpyHostToDevice) != cudaSuccess) *ok = false;
  return (const Tp*)d;
}

#include "omg_sp_host.cuh"

// pack a term list into 32-byte records; aux = lrow (W) / slot offset within the row (J)
static const PTerm* upload_terms(omg_problem* h, const omg_termlist& L, int n_one,
                                 const std::vector<int>* aux, bool* ok) {
  std::vector<PTerm> pk((size_t)L.n_terms + 1);
  memset(pk.data(), 0, pk.size() * sizeof(PTerm));
  for (int k = 0; k < L.n_terms; ++k) {
    PTerm& q = pk[k];
    q.coef = L.coef[k]; q.cidx = (unsigned short)L.cidx[k];
    q.aux = (unsigned short)(aux ? (*aux)[k] : (L.lrow ? L.lrow[k] : 0));
    for (int w = 0; w < MAXW; ++w)
      q.x[w] = (unsigned short)(w < L.width ? L.xi[(size_t)k * L.width + w] : n_one);
  }
  for (int w = 0; w < MAXW; ++w) pk[L.n_terms].x[w] = (unsigned short)n_one;
  return upload(h, pk.data(), pk.size(), ok);
}

extern "C" {

int omg_abi_version(void) { return OMG_ABI_VERSION; }
#ifdef OMG_CPU_EMU
// only the CPU emulation build (tools/cpu_emu) exports this: its "device" pointers are host
// pointers, which lets the tests drive the device-pointer API with CPU tensors
int omg_is_emulation(void) { return 1; }
#endif

// ---- table files ---------------------------------------------------------------
namespace {
struct TabField { const char* name; int dtype; size_t off; int scalar; };
#define TF_S(f)      {#f, 0, offsetof(omg_tables, f), 1}
#define TF_I(f)      {#f, 0, offsetof(omg_tables, f), 0}
#define TF_D(f)      {#f, 1, offsetof(omg_tables, f), 0}
#define TF_LS(l, f)  {#l "." #f, 0, offsetof(omg_tables, l) + offsetof(omg_termlist, f), 1}
#define TF_LI(l, f)  {#l "." #f, 0, offsetof(omg_tables, l) + offsetof(omg_termlist, f), 0}
#define TF_LD(l, f)  {#l "." #f, 1, offsetof(omg_tables, l) + offsetof(omg_termlist, f), 0}
#define TF_LIST(l)   TF_LS(l, n_out), TF_LS(l, n_terms), TF_LS(l, width), TF_LI(l, ptr), TF_LD(l, coef), \
                     TF_LI(l, cidx), TF_LI(l, xi), TF_LI(l, lrow)
const TabField kTabFields[] = {
  TF_S(n), TF_S(m), TF_S(n_par), TF_S(n_v), TF_S(degree), TF_S(n_tape), TF_S(n_tape_terms), TF_S(n_levels),
  TF_I(tape_func), TF_I(tape_ptr), TF_D(tape_coef), TF_I(tape_fac), TF_I(level_ptr),
  TF_LIST(G), TF_LIST(F), TF_LIST(DF), TF_LIST(J), TF_LIST(W),
  TF_S(nnz_j), TF_I(jrow), TF_I(jcol), TF_I(jrow_ptr),
  TF_S(n_mid), TF_S(nnz_jx), TF_S(n_jp), TF_S(n_mu), TF_I(jp_ptr), TF_I(jp_a), TF_I(jp_c),
  TF_I(mu_ptr), TF_I(mu_row), TF_I(mu_slot),
  TF_S(nnz_w), TF_I(wrow), TF_I(wcol), TF_I(w2h),
  TF_S(nnz_h), TF_S(n_hp), TF_I(hrow), TF_I(hcol), TF_I(hp_ptr), TF_I(hp_s1), TF_I(hp_s2), TF_I(hp_row),
  TF_D(lbg), TF_D(ubg),
  TF_S(kkt_n), TF_S(kkt_n_eq), TF_S(env_size), TF_S(n_panel_rows), TF_S(max_panel_rows),
  TF_I(kkt_eq_rows), TF_I(kkt_pos_var), TF_I(kkt_pos_eq), TF_I(kkt_sign), TF_I(env_first), TF_I(env_ptr),
  TF_I(kkt_hdst), TF_I(kkt_jdst), TF_I(kkt_diag), TF_I(kkt_panel_ptr), TF_I(kkt_panel_rows),
  TF_S(nnz_wx), TF_S(n_xq), TF_S(n_xp), TF_I(xq_h), TF_I(xq_ptr), TF_I(xq_w), TF_I(xq_a), TF_I(xq_b),
};
struct OwnedTables { omg_tables T; std::vector<void*> blocks; };
}  // namespace

omg_tables* omg_tables_read(const char* path) {
  FILE* fp = path ? fopen(path, "rb") : nullptr;
  if (!fp) { set_err(std::string("cannot open table file ") + (path ? path : "(null)")); return nullptr; }
  OwnedTables* O = new OwnedTables();
  memset(&O->T, 0, sizeof(O->T));
  bool ok = true;
  char magic[8]; int32_t ver = 0, nrec = 0;
  if (fread(magic, 1, 8, fp) != 8 || memcmp(magic, "OMGTBL\0\0", 8) != 0) { set_err("not an omg table file"); ok = false; }
  if (ok && (fread(&ver, 4, 1, fp) != 1 || fread(&nrec, 4, 1, fp) != 1)) { set_err("truncated table file"); ok = false; }
  if (ok && ver != OMG_ABI_VERSION) { set_err("table file written for another ABI version"); ok = false; }
  O->T.abi_version = ver;
  const int nf = (int)(sizeof(kTabFields) / sizeof(kTabFields[0]));
  std::vector<char> seen(nf, 0);
  for (int r = 0; ok && r < nrec; ++r) {
    char name[24]; int32_t dtype = 0, pad = 0; int64_t count = 0;
    if (fread(name, 1, 24, fp) != 24 || fread(&dtype, 4, 1, fp) != 1 || fread(&pad, 4, 1, fp) != 1 ||
        fread(&count, 8, 1, fp) != 1 || count < 0) { set_err("truncated table file"); ok = false; break; }
    name[23] = 0;
    int k = -1;
    for (int q = 0; q < nf; ++q) if (strcmp(kTabFields[q].name, name) == 0) { k = q; break; }
    const size_t esz = dtype ? 8 : 4;
    if (k < 0 || kTabFields[k].dtype != dtype) { set_err(std::string("unknown record in table file: ") + name); ok = false; break; }
    char* base = reinterpret_cast<char*>(&O->T) + kTabFields[k].off;
    if (kTabFields[k].scalar) {
      if (count != 1 || fread(base, 4, 1, fp) != 1) { set_err("bad scalar record"); ok = false; break; }
    } else {
      void* blk = malloc((size_t)(count > 0 ? count : 1) * esz);
      O->blocks.push_back(blk);
      if (!blk || (count > 0 && fread(blk, esz, (size_t)count, fp) != (size_t)count)) { set_err("truncated table file"); ok = false; break; }
      *reinterpret_cast<void**>(base) = (count > 0 || strcmp(name + strlen(name) - 4, "lrow") != 0) ? blk : nullptr;
    }
    seen[k] = 1;
  }
  fclose(fp);
  // lrow of the lists without multipliers is legitimately absent; everything else is required
  for (int q = 0; ok && q < nf; ++q)
    if (!seen[q] && !strstr(kTabFields[q].name, ".lrow")) { set_err(std::string("table file lacks ") + kTabFields[q].name); ok = false; }
  if (!ok) { omg_tables_free(&O->T); return nullptr; }
  return &O->T;
}

void omg_tables_free(omg_tables* tables) {
  if (!tables) return;
  OwnedTables* O = reinterpret_cast<OwnedTables*>(tables);   // T is the first member
  for (void* b : O->blocks) free(b);
  delete O;
}
const char* omg_last_error(void) { return g_err.c_str(); }

void omg_default_options(omg_options* o) {
  o->tol = 1e-3; o->constr_viol_tol = 1e-4; o->dual_inf_tol = 1.0; o->compl_inf_tol = 1e-4;
  o->mu_init = 0.1; o->bound_push = 1e-3; o->bound_frac = 1e-3; o->mult_bound_push = 1e-3;
  o->bound_relax_factor = 1e-8; o->scaling_max_gradient = 100.0;
  o->max_iter = 3000; o->trace = 0;
  o->max_restarts = 5; o->soft_resto = 1; o->restart_mu = 1.0; o->restart_push = 0.1;
  o->inertia_mode = 0; o->reserved = 0;
}

omg_problem* omg_problem_create(const omg_tables* tb, const omg_options* opt, int device) {
  if (!tb || tb->abi_version != OMG_ABI_VERSION) { set_err("omg_tables ABI version mismatch"); return nullptr; }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    set_err("no CUDA device available: libomgb200 has no CPU fallback"); return nullptr; }
  if (device < 0 || device >= ndev) { set_err("invalid device index"); return nullptr; }
  if (cudaSetDevice(device) != cudaSuccess) { set_err("cudaSetDevice failed"); return nullptr; }
  g_err.clear();
  omg_problem* h = new omg_problem();
  h->device = device;
  if (opt) h->opt = *opt; else omg_default_options(&h->opt);
  bool ok = true;
  DevTab& T = h->T;
  memset(&T, 0, sizeof(T));
  const int n = tb->n, m = tb->m;
  T.n = n; T.m = m; T.n_par = tb->n_par; T.n_v = tb->n_v;
  T.n_tape = tb->n_tape; T.n_levels = tb->n_levels;
  T.nnz_j = tb->nnz_j; T.nnz_w = tb->nnz_w; T.nnz_h = tb->nnz_h;
  T.n_eq = tb->kkt_n_eq; T.N = tb->kkt_n;
  T.env_size = tb->env_size; T.max_panel_rows = tb->max_panel_rows;
  T.n_panel_rows = tb->n_panel_rows;
  T.n_panels = (tb->kkt_n + NB - 1) / NB;
  if (tb->kkt_n != n + tb->kkt_n_eq) { set_err("inconsistent KKT structure"); ok = false; }
  const int n_mid = tb->n_mid;
  T.n_mid = n_mid; T.nnz_jx = n_mid ? tb->nnz_jx : tb->nnz_j;
  if (!(n + 1 + n_mid < 65535 && tb->n_v < 65536 && m + 1 + n_mid < 65535 && tb->nnz_j < 65536)) {
    set_err("problem too large for 16-bit packed indices"); ok = false; }
  const omg_termlist* lists[5] = {&tb->G, &tb->F, &tb->DF, &tb->J, &tb->W};
  for (int k = 0; k < 5 && ok; ++k)
    if (lists[k]->width > MAXW) { set_err("term degree exceeds the record width (5 factors)"); ok = false; }
  for (int i = 0; ok && i <= tb->kkt_n; ++i)
    if (tb->env_first[i] % NB != 0) {
      set_err("envelope rows must start at multiples of the panel width"); ok = false; }
  if (!ok) { delete h; return nullptr; }

  h->lbg = upload(h, tb->lbg, m, &ok);
  h->ubg = upload(h, tb->ubg, m, &ok);
  T.tape_func = upload(h, tb->tape_func, tb->n_tape, &ok);
  T.tape_ptr = upload(h, tb->tape_ptr, (size_t)tb->n_tape + 1, &ok);
  T.tape_coef = upload(h, tb->tape_coef, tb->n_tape_terms, &ok);
  T.tape_fac = upload(h, tb->tape_fac, (size_t)tb->n_tape_terms * 4, &ok);
  T.level_ptr = upload(h, tb->level_ptr, (size_t)tb->n_levels + 1, &ok);
  // term records
  T.Gt = upload_terms(h, tb->G, n, nullptr, &ok);
  T.Ft = upload_terms(h, tb->F, n, nullptr, &ok); T.n_f = tb->F.n_terms;
  T.DFt = upload_terms(h, tb->DF, n, nullptr, &ok);
  T.dfptr = upload(h, tb->DF.ptr, (size_t)n + 1, &ok);
  T.Wt = upload_terms(h, tb->W, n, nullptr, &ok);
  {
    std::vector<int> aux(tb->J.n_terms > 0 ? tb->J.n_terms : 1);
    for (int s = 0; s < tb->nnz_j; ++s) {
      const int off = s - tb->jrow_ptr[tb->jrow[s]];
      for (int t = tb->J.ptr[s]; t < tb->J.ptr[s + 1]; ++t) aux[t] = off;
    }
    T.Jt = upload_terms(h, tb->J, n, &aux, &ok);
  }
  {  // per-row records
    std::vector<RowRec> rr(m > 0 ? m : 1);
    for (int i = 0; i < m; ++i) {
      RowRec& r = rr[i];
      r.g0 = tb->G.ptr[i]; r.g1 = tb->G.ptr[i + 1];
      r.s0 = tb->jrow_ptr[i]; r.ns = tb->jrow_ptr[i + 1] - tb->jrow_ptr[i];
      r.jt0 = tb->J.ptr[r.s0]; r.jt1 = tb->J.ptr[r.s0 + r.ns];
      r.pad0 = r.pad1 = 0;
      // every slot of the row must own at least one term (aux bookkeeping); with
      // intermediates the chain-rule pass initialises every slot instead
      for (int s = r.s0; s < r.s0 + r.ns && !n_mid; ++s)
        if (tb->J.ptr[s + 1] == tb->J.ptr[s]) { set_err("empty Jacobian slot"); ok = false; }
    }
    T.rowrec = upload(h, rr.data(), rr.size(), &ok);
  }
  if (n_mid) {  // intermediates: term ranges and chain-rule lists
    std::vector<int2> mg(n_mid);
    for (int l = 0; l < n_mid; ++l) mg[l] = make_int2(tb->G.ptr[m + l], tb->G.ptr[m + l + 1]);
    T.midg = upload(h, mg.data(), mg.size(), &ok);

    T.jp_ptr = upload(h, tb->jp_ptr, (size_t)tb->nnz_j + 1, &ok);
    T.jp_a = upload(h, tb->jp_a, tb->n_jp, &ok);
    T.jp_c = upload(h, tb->jp_c, tb->n_jp, &ok);
    T.mu_ptr = upload(h, tb->mu_ptr, (size_t)n_mid + 1, &ok);
    T.mu_row = upload(h, tb->mu_row, tb->n_mu, &ok);
    T.mu_slot = upload(h, tb->mu_slot, tb->n_mu, &ok);
    std::vector<int> xv;   // extra slots with at least one x factor (xi != n, the constant 1)
    for (int s = tb->nnz_j; s < tb->nnz_jx; ++s) {
      bool dep = false;
      for (int t = tb->J.ptr[s]; t < tb->J.ptr[s + 1] && !dep; ++t)
        for (int w = 0; w < tb->J.width; ++w) if (tb->J.xi[(size_t)t * tb->J.width + w] != n) { dep = true; break; }
      if (dep) xv.push_back(s);
    }
    T.n_jxvar = (int)xv.size();
    if (xv.empty()) xv.push_back(0);
    T.jxvar = upload(h, xv.data(), xv.size(), &ok);
  }
  T.jtptr = upload(h, tb->J.ptr, (size_t)T.nnz_jx + 1, &ok);
  T.jrow = upload(h, tb->jrow, tb->nnz_j, &ok);
  {  // CSC view of the Jacobian pattern: slot | row << 16
    std::vector<int> cptr(n + 1, 0);
    std::vector<unsigned> crec(tb->nnz_j > 0 ? tb->nnz_j : 1);
    std::vector<unsigned short> jc(tb->nnz_j > 0 ? tb->nnz_j : 1);
    for (int s = 0; s < tb->nnz_j; ++s) { cptr[tb->jcol[s] + 1]++; jc[s] = (unsigned short)tb->jcol[s]; }
    for (int j = 0; j < n; ++j) cptr[j + 1] += cptr[j];
    std::vector<int> fill(cptr.begin(), cptr.end() - 1);
    for (int s = 0; s < tb->nnz_j; ++s)
      crec[fill[tb->jcol[s]]++] = (unsigned)s | ((unsigned)tb->jrow[s] << 16);
    T.colptr = upload(h, cptr.data(), cptr.size(), &ok);
    T.colrec = upload(h, crec.data(), crec.size(), &ok);
    T.jcol16 = upload(h, jc.data(), jc.size(), &ok);
  }
  {  // H positions sorted by descending pair count (balanced warps) + packed pairs
    std::vector<int> order(tb->nnz_h);
    for (int q = 0; q < tb->nnz_h; ++q) order[q] = q;
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) {
      return (tb->hp_ptr[a + 1] - tb->hp_ptr[a]) > (tb->hp_ptr[b + 1] - tb->hp_ptr[b]); });
    std::vector<HqRec> hq(tb->nnz_h > 0 ? tb->nnz_h : 1);
    std::vector<unsigned> pack((size_t)tb->n_hp + 1);
    int pos = 0;
    std::vector<char> has(n, 0);
    for (int k = 0; k < tb->nnz_h; ++k) {
      const int q = order[k];
      HqRec& r = hq[k];
      r.dst = tb->kkt_hdst[q]; r.p0 = pos; r.diag = (tb->hrow[q] == tb->hcol[q]) ? 1 : 0;
      if (r.diag) has[tb->hrow[q]] = 1;
      for (int e = tb->hp_ptr[q]; e < tb->hp_ptr[q + 1]; ++e)
        pack[pos++] = (unsigned)tb->hp_s1[e] | ((unsigned)tb->hp_s2[e] << 16);
      r.p1 = pos;
      if (r.p1 - r.p0 >= 64) T.n_hq_heavy = k + 1;
    }
    for (int j = 0; j < n; ++j) if (!has[j]) {
      set_err("H pattern lacks a diagonal entry (variable without constraint)"); ok = false; break; }
    T.hq = upload(h, hq.data(), hq.size(), &ok);
    T.hpack = upload(h, pack.data(), pack.size(), &ok);
  }
  const int nnz_wx = n_mid ? tb->nnz_wx : 0;
  T.nnz_wx = nnz_wx; T.n_xq = nnz_wx ? tb->n_xq : 0;
  if (tb->W.n_out != tb->nnz_w + nnz_wx) { set_err("W term list does not match nnz_w + nnz_wx"); ok = false; }
  if (ok) {  // Hessian slots: destination in the envelope (cross slots: index into Wx) + term range
    std::vector<WRec> wr(tb->nnz_w + nnz_wx > 0 ? tb->nnz_w + nnz_wx : 1);
    for (int q = 0; q < tb->nnz_w + nnz_wx; ++q) {
      wr[q].dst = (q < tb->nnz_w) ? tb->kkt_hdst[tb->w2h[q]] : q - tb->nnz_w;
      wr[q].t0 = tb->W.ptr[q]; wr[q].t1 = tb->W.ptr[q + 1]; wr[q].pad = 0;
    }
    T.wrec = upload(h, wr.data(), wr.size(), &ok);
  }
  if (ok && nnz_wx) {  // cross-Hessian gather records
    std::vector<HqRec> xq(T.n_xq > 0 ? T.n_xq : 1);
    std::vector<int4> xp(tb->n_xp > 0 ? tb->n_xp : 1);
    for (int e = 0; e < T.n_xq && ok; ++e) {
      const int q = tb->xq_h[e];
      if (q < 0 || q >= tb->nnz_h) { set_err("cross-Hessian position out of range"); ok = false; break; }
      xq[e].dst = tb->kkt_hdst[q]; xq[e].p0 = tb->xq_ptr[e]; xq[e].p1 = tb->xq_ptr[e + 1];
      xq[e].diag = (tb->hrow[q] == tb->hcol[q]) ? 1 : 0;
    }
    for (int r = 0; r < tb->n_xp && ok; ++r) {
      const int a = tb->xq_a[r], b = tb->xq_b[r];
      if (tb->xq_w[r] < 0 || tb->xq_w[r] >= nnz_wx || a < tb->nnz_j || a >= tb->nnz_jx ||
          (b >= 0 && (b < tb->nnz_j || b >= tb->nnz_jx))) {
        set_err("extra Hessian product out of range"); ok = false; break; }
      xp[r] = make_int4(tb->xq_w[r], a, b, 0);
    }
    T.xq = upload(h, xq.data(), xq.size(), &ok);
    T.xqp = upload(h, xp.data(), xp.size(), &ok);
  }
  T.eq_rows = upload(h, tb->kkt_eq_rows, tb->kkt_n_eq, &ok);
  T.pos_var = upload(h, tb->kkt_pos_var, n, &ok);
  T.pos_eq = upload(h, tb->kkt_pos_eq, tb->kkt_n_eq, &ok);
  T.ksign = upload(h, tb->kkt_sign, tb->kkt_n, &ok);
  T.env_first = upload(h, tb->env_first, (size_t)tb->kkt_n + 1, &ok);
  T.env_ptr = upload(h, tb->env_ptr, (size_t)tb->kkt_n + 2, &ok);
  T.jdst = upload(h, tb->kkt_jdst, tb->nnz_j, &ok);
  T.kdiag = upload(h, tb->kkt_diag, tb->kkt_n, &ok);
  T.panel_ptr = upload(h, tb->kkt_panel_ptr, (size_t)T.n_panels + 1, &ok);
  T.panel_rows = upload(h, tb->kkt_panel_rows, tb->n_panel_rows, &ok);
  {
    std::vector<int> cmin(T.n_panels > 0 ? T.n_panels : 1);
    for (int pb = 0; pb < T.n_panels; ++pb) {
      int c = pb * NB;
      for (int r = pb * NB; r < tb->kkt_n && r < (pb + 1) * NB; ++r) c = tb->env_first[r] < c ? tb->env_first[r] : c;
      cmin[pb] = c;
    }
    T.panel_cmin = upload(h, cmin.data(), cmin.size(), &ok);
  }

  // ---- shared-memory layout: mandatory part, then per-instance arrays by priority
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) ok = false;
  h->n_sm = prop.multiProcessorCount;
  Smem& S = h->S;
  const int N = T.N;
  int off = 0;
  auto take = [&](int cnt) { int o = off; off += (cnt + 1) & ~1; return o; };
  const int xe_len = n + 1 + n_mid;
  // mandatory shared-memory part; K and the parameter tape V optionally in scratch
  auto layout = [&](bool k_smem, bool v_smem) {
    off = 0;
    S.K = k_smem ? take(T.env_size + 2) : -1;
    S.LDP = (T.max_panel_rows + 2 + 3) & ~3;
    S.Pt = take(NB * S.LDP); S.PtS = take(NB * S.LDP); S.Ld = take(NB * NB);
    S.rbase = take(S.LDP);               // 2*LDP ints: row base offsets + row ids
    S.xe = take(xe_len); S.xt = take(xe_len); S.dx = take(N + 1); S.u = take(N + 1);
    S.gf = take(n);
    S.diag0 = take(N + 1); S.invd = take(N + 1); S.V = v_smem ? take(T.n_v) : -1;
    S.red = take(MAX_NWARP * NRED); S.filt = take(2 * MAXF);
    S.rt8 = take((m + 7) / 8);
    S.sgn = take(N); S.eptr = take((N + 2 + 1) / 2); S.efirst = take((N + 1 + 1) / 2);
    S.pptr = take((T.n_panels + 1 + 1) / 2); S.prow = take((tb->n_panel_rows + 1) / 2);
    S.pcmin = take((T.n_panels + 1) / 2);
    return (size_t)off * 8;
  };
  // standard kernels keep K and V in shared memory; the XL kernel (intermediates, or a
  // structure too large for that) keeps V in scratch, and K too if it leaves no room
  bool k_in_smem = true;
  {
    cudaFuncAttributes f0, fx;
    size_t b0 = 0, bx = 0;
    if (cudaFuncGetAttributes(&f0, (const void*)omg_ipm_kernel<false>) == cudaSuccess)
      b0 = (size_t)prop.sharedMemPerBlockOptin - f0.sharedSizeBytes;
    if (cudaFuncGetAttributes(&fx, (const void*)omg_ipm_kernel_xl<false>) == cudaSuccess)
      bx = (size_t)prop.sharedMemPerBlockOptin - fx.sharedSizeBytes;
    h->xl = (n_mid > 0) || layout(true, true) > b0;
    if (h->xl) {
      // what is read at random stays on the SM in this order: K, then the parameter tape V (one
      // load per TERM of every stream); the m-vectors are streamed one thread per row and go last
      if (layout(true, true) <= bx) { }
      else if (layout(true, false) <= bx) { }
      else { k_in_smem = false; if (layout(false, true) > bx) layout(false, false); }
    } else layout(true, true);
  }
  // blocks per SM: 2 x 256 threads overlap one block's serial pivots with the other's
  // parallel phases; 1 x 512 keeps every per-instance array in shared memory.
  cudaFuncAttributes fa;
  if (ok && cudaFuncGetAttributes(&fa, h->xl ? (const void*)omg_ipm_kernel_xl<false> : (const void*)omg_ipm_kernel<false>) != cudaSuccess) { set_err("cudaFuncGetAttributes failed"); ok = false; }
  const size_t budget1 = ok ? (size_t)prop.sharedMemPerBlockOptin - fa.sharedSizeBytes : 0;
  const size_t budget2 = ok ? ((size_t)prop.sharedMemPerMultiprocessor - 2 * 1024) / 2 - fa.sharedSizeBytes : 0;
  {
    const char* e = getenv("OMG_B200_CTAS");
    const int want = (e && atoi(e) == 1) ? 1 : 2;
    h->target_ctas = (want == 2 && (!h->xl || !k_in_smem) && (size_t)off * 8 <= budget2) ? 2 : 1;
    h->nt = (h->target_ctas == 1) ? 512 : 256;
  }
  h->wide = T.max_panel_rows + 2 > h->nt;   // panels reach more rows than the block has threads
  const void* kfn = h->wide ? (h->xl ? ((h->target_ctas == 1) ? (const void*)omg_ipm_kernel_xl<true> : (const void*)omg_ipm_kernel_xl_2cta<true>)
                                     : (h->target_ctas == 1) ? (const void*)omg_ipm_kernel<true> : (const void*)omg_ipm_kernel_2cta<true>)
                            : (h->xl ? ((h->target_ctas == 1) ? (const void*)omg_ipm_kernel_xl<false> : (const void*)omg_ipm_kernel_xl_2cta<false>)
                                     : (h->target_ctas == 1) ? (const void*)omg_ipm_kernel<false> : (const void*)omg_ipm_kernel_2cta<false>);
  const size_t budget = (h->target_ctas == 1) ? budget1 : budget2;
  if (ok && (size_t)off * 8 > budget) {
    char buf[256];
    snprintf(buf, sizeof buf, "KKT envelope does not fit shared memory: need %zu B, have %zu B (n=%d, n_eq=%d)",
             (size_t)off * 8, budget, n, T.n_eq);
    set_err(buf); ok = false;
  }
  int goff = 0;   // global scratch offset (doubles)
  S.Kg = S.Vg = S.jxg = S.mug = S.Kcg = S.wxg = 0;
  if (h->xl) {
    auto gtake = [&](int cnt) { int o = goff; goff += (cnt + 1) & ~1; return o; };
    S.Vg = gtake(T.n_v);
    S.jxg = gtake(T.nnz_jx - T.nnz_j + 1);
    S.mug = gtake(n_mid + 1);
    S.wxg = gtake(T.nnz_wx + 1);
    if (!k_in_smem) S.Kg = gtake(T.env_size + 2);
  }
  S.Kcg = goff; goff += (T.env_size + 2 + 1) & ~1;
  const int sizes[N_ARR] = {tb->nnz_j, m, tb->nnz_j, m, m, m, m, m, m, m, m, m, m, m, m, m, m, m, m};
  for (int k = 0; k < N_ARR; ++k) {
    const int cnt = (sizes[k] + 1) & ~1;
    const bool optional_low = (k >= A_ZL);     // lower-bound / equality-only arrays: rarely touched
    if (!optional_low && (size_t)(off + cnt) * 8 <= budget) { S.arr[k] = off; off += cnt; }
    else { S.arr[k] = -(goff + 1); goff += cnt; }
  }
  S.total = off;
  h->smem_bytes = (size_t)off * sizeof(double);
  if (ok && cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)((size_t)prop.sharedMemPerBlockOptin - fa.sharedSizeBytes)) != cudaSuccess) {
    set_err(std::string("cudaFuncSetAttribute failed: ") + cudaGetErrorString(cudaGetLastError())); ok = false; }
  if (ok) {
    int occ = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kfn, h->nt, h->smem_bytes);
    h->ctas_per_sm = occ > 0 ? occ : 1;
    h->dscr_stride = goff + 8;
    h->iscr_stride = 2 * m + 8;
    {  // sparse variant: preferred whenever the problem is inside its coverage
      const char* e = getenv("OMG_B200_KERNEL");   // "envelope": force the envelope kernels
      std::string why;
      h->env_nt = h->nt; h->env_ctas = h->ctas_per_sm; h->env_smem_bytes = h->smem_bytes;
      {  // the envelope kernels' layout (they run inertia_mode = 1 and what the sparse kernel
         // rejects); min-panel-rows leaves out the last panel, which reaches only the
         // right-hand-side row
        int arr_scratch = 0;
        for (int k = 0; k < N_ARR; ++k) arr_scratch += (S.arr[k] < 0) ? 1 : 0;
        int min_rows = tb->kkt_panel_ptr[1] - tb->kkt_panel_ptr[0];
        for (int pb = 1; pb + 1 < T.n_panels; ++pb)
          min_rows = std::min(min_rows, tb->kkt_panel_ptr[pb + 1] - tb->kkt_panel_ptr[pb]);
        h->env_info = std::string("kernel=") + (h->xl ? "xl" : "standard") + " nt=" + std::to_string(h->env_nt) +
                      " K=" + (S.K >= 0 ? "shared" : "scratch") + " V=" + (S.V >= 0 ? "shared" : "scratch") +
                      " arrays-in-scratch=" + std::to_string(arr_scratch) +
                      " max-panel-rows=" + std::to_string(T.max_panel_rows) +
                      " min-panel-rows=" + std::to_string(min_rows) + " N%8=" + std::to_string(N % NB) +
                      " wide=" + (h->wide ? "1" : "0");
      }
      if (!(e && strcmp(e, "envelope") == 0) && sp_setup(h, tb, prop, &why)) {
        h->sp = true;
        h->nt = h->P.nt; h->ctas_per_sm = h->sp_ctas;
        h->smem_bytes = h->sp_smem_bytes;
        if (h->sp_dscr_stride > h->dscr_stride) h->dscr_stride = h->sp_dscr_stride;
      } else h->sp_info = "envelope kernels (" + (why.empty() ? std::string("forced") : why) + ")";
      if (getenv("OMG_B200_VERBOSE")) {
        fprintf(stderr, "[omg_b200] %s\n", h->sp_info.c_str());
        if (!h->sp) {   // what the sparse ordering would give on this structure (diagnostic only)
          SpSym Y; std::string w2;
          const bool sy = sp_symbolic(tb, Y, &w2);
          int pairs = 0;
          for (int j = 0; j < Y.R0 && j < (int)Y.st.size(); ++j) pairs += (int)(Y.st[j].size() * (Y.st[j].size() + 1) / 2);
          fprintf(stderr, "[omg_b200]   symbolic (%s): N=%d Lsize=%d levels=%d root=%d pairs(non-root)=%d env_size=%d\n",
                  sy ? "ok" : w2.c_str(), Y.N, Y.Lsize, Y.n_lev, Y.nr, pairs, T.env_size);
        }
      }
    }
    if (cudaMalloc(&h->counter, sizeof(int)) != cudaSuccess) ok = false;
    if (cudaMalloc(&h->trace, sizeof(double) * TRACE_ROWS * TRACE_COLS) != cudaSuccess) ok = false;
    else cudaMemset(h->trace, 0, sizeof(double) * TRACE_ROWS * TRACE_COLS);
    cudaEventCreate(&h->ev0); cudaEventCreate(&h->ev1);
  }
  if (!ok) { if (g_err.empty()) set_err("device allocation/upload failed"); omg_problem_destroy(h); return nullptr; }
  return h;
}

void omg_problem_destroy(omg_problem* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  for (void* p : h->allocs) cudaFree(p);
  if (h->dscr) cudaFree(h->dscr);
  if (h->iscr) cudaFree(h->iscr);
  if (h->fscr) cudaFree(h->fscr);
  free_desc(h->shift_desc);
  if (h->counter) cudaFree(h->counter);
  if (h->trace) cudaFree(h->trace);
  if (h->ev0) cudaEventDestroy(h->ev0);
  if (h->ev1) cudaEventDestroy(h->ev1);
  void* st[] = {h->hx0, h->hp, h->hlb, h->hub, h->hlam0, h->hx, h->hlam, h->hf, h->hst, h->hit};
  for (void* p : st) if (p) cudaFree(p);
  delete h;
}

int omg_set_options(omg_problem* h, const omg_options* opt) {
  if (!h || !opt) { set_err("null argument"); return -1; }
  h->opt = *opt; return 0;
}

int omg_get_info(omg_problem* h, int32_t* n, int32_t* m, int32_t* n_par, int32_t* smem_bytes,
                 int32_t* ctas_per_sm, int32_t* n_sm) {
  if (!h) { set_err("null handle"); return -1; }
  if (n) *n = h->T.n; if (m) *m = h->T.m; if (n_par) *n_par = h->T.n_par;
  if (smem_bytes) *smem_bytes = (int32_t)h->smem_bytes;
  if (ctas_per_sm) *ctas_per_sm = h->ctas_per_sm; if (n_sm) *n_sm = h->n_sm;
  return 0;
}

const char* omg_structure_info(omg_problem* h) { return h ? h->sp_info.c_str() : ""; }
const char* omg_envelope_layout(omg_problem* h) { return h ? h->env_info.c_str() : ""; }

}  // extern "C"

// omg_solve_batch on the rows listed in DEVICE rows [*n_rows] (ascending; both null: every row).
// The grid is min(B, resident blocks) whatever the list holds, so the launch shape does not
// depend on device data; an unlisted row's outputs are not written.
static int solve_batch_rows(omg_problem* h, int32_t B, const double* x0, const double* p,
                            const double* lbg, const double* ubg, int32_t bounds_shared,
                            const double* lam_g0, double* x, double* lam_g, double* f,
                            int32_t* status, int32_t* iters, const int* rows, const int* n_rows,
                            void* stream_) {
  if (!h) { set_err("null handle"); return -1; }
  if (B <= 0) return 0;
  if (!x0 || !p || !lbg || !ubg || !x || !lam_g || !f || !status || !iters) { set_err("null buffer"); return -1; }
  cudaStream_t stream = (cudaStream_t)stream_;
  CK(cudaSetDevice(h->device));
  const bool use_sp = h->sp && h->opt.inertia_mode == 0;
  int grid = h->n_sm * (use_sp ? h->sp_ctas : h->env_ctas);
  if (grid > B) grid = B;
  if (grid > h->scr_ctas) {
    if (h->dscr) cudaFree(h->dscr);
    if (h->iscr) cudaFree(h->iscr);
    h->dscr = nullptr; h->iscr = nullptr;
    const int want = h->n_sm * std::max(h->ctas_per_sm, h->env_ctas);
    CK(cudaMalloc(&h->dscr, (size_t)want * h->dscr_stride * sizeof(double)));
    CK(cudaMalloc(&h->iscr, (size_t)want * h->iscr_stride * sizeof(int)));
    h->scr_ctas = want;
  }
  Batch A;
  A.B = B; A.bounds_shared = bounds_shared;
  A.x0 = x0; A.p = p; A.lbg = lbg; A.ubg = ubg; A.lam0 = lam_g0;
  A.x = x; A.lam = lam_g; A.f = f; A.status = status; A.iters = iters;
  A.dscr = h->dscr; A.iscr = h->iscr; A.dscr_stride = h->dscr_stride; A.iscr_stride = h->iscr_stride;
  A.counter = h->counter; A.trace = h->trace;
  A.rows = rows; A.n_rows = n_rows;
  CK(cudaMemsetAsync(h->counter, 0, sizeof(int), stream));
  CK(cudaEventRecord(h->ev0, stream));
  if (use_sp) OMG_LAUNCH(omg_ipm_kernel_sp, grid, h->P.nt, h->sp_smem_bytes, stream, h->T, h->P, h->opt, A, h->SS);
  else if (h->wide) {
    if (h->xl && h->target_ctas == 1) OMG_LAUNCH(omg_ipm_kernel_xl<true>, grid, 512, h->env_smem_bytes, stream, h->T, h->opt, A, h->S);
    else if (h->xl) OMG_LAUNCH(omg_ipm_kernel_xl_2cta<true>, grid, 256, h->env_smem_bytes, stream, h->T, h->opt, A, h->S);
    else if (h->target_ctas == 1) OMG_LAUNCH(omg_ipm_kernel<true>, grid, 512, h->env_smem_bytes, stream, h->T, h->opt, A, h->S);
    else OMG_LAUNCH(omg_ipm_kernel_2cta<true>, grid, 256, h->env_smem_bytes, stream, h->T, h->opt, A, h->S);
  }
  else if (h->xl && h->target_ctas == 1) OMG_LAUNCH(omg_ipm_kernel_xl<false>, grid, 512, h->env_smem_bytes, stream, h->T, h->opt, A, h->S);
  else if (h->xl) OMG_LAUNCH(omg_ipm_kernel_xl_2cta<false>, grid, 256, h->env_smem_bytes, stream, h->T, h->opt, A, h->S);
  else if (h->target_ctas == 1) OMG_LAUNCH(omg_ipm_kernel<false>, grid, 512, h->env_smem_bytes, stream, h->T, h->opt, A, h->S);
  else OMG_LAUNCH(omg_ipm_kernel_2cta<false>, grid, 256, h->env_smem_bytes, stream, h->T, h->opt, A, h->S);
  CK(cudaGetLastError());
  CK(cudaEventRecord(h->ev1, stream));
  h->timed = true; h->launches = 1;
  return 0;
}

extern "C" {

int omg_solve_batch(omg_problem* h, int32_t B, const double* x0, const double* p,
                    const double* lbg, const double* ubg, int32_t bounds_shared,
                    const double* lam_g0, double* x, double* lam_g, double* f,
                    int32_t* status, int32_t* iters, void* stream_) {
  return solve_batch_rows(h, B, x0, p, lbg, ubg, bounds_shared, lam_g0, x, lam_g, f, status, iters, nullptr,
                          nullptr, stream_);
}

int omg_solve_batch_rows(omg_problem* h, int32_t B, const double* x0, const double* p,
                         const double* lbg, const double* ubg, int32_t bounds_shared,
                         const double* lam_g0, double* x, double* lam_g, double* f,
                         int32_t* status, int32_t* iters, const int32_t* rows, const int32_t* n_rows,
                         void* stream_) {
  if (!rows || !n_rows) { set_err("omg_solve_batch_rows: null row list"); return -1; }
  return solve_batch_rows(h, B, x0, p, lbg, ubg, bounds_shared, lam_g0, x, lam_g, f, status, iters, rows, n_rows,
                          stream_);
}

int omg_last_timing(omg_problem* h, float* kernel_ms, int32_t* launches) {
  if (!h || !h->timed) { set_err("no solve recorded"); return -1; }
  CK(cudaEventSynchronize(h->ev1));
  float ms = 0.f;
  CK(cudaEventElapsedTime(&ms, h->ev0, h->ev1));
  if (kernel_ms) *kernel_ms = ms;
  if (launches) *launches = h->launches;
  return 0;
}

int omg_get_trace(omg_problem* h, double* out, int32_t max_rows) {
  if (!h || !out) { set_err("null argument"); return -1; }
  CK(cudaSetDevice(h->device));
  CK(cudaDeviceSynchronize());
  int rows = max_rows < TRACE_ROWS ? max_rows : TRACE_ROWS;
  CK(cudaMemcpy(out, h->trace, sizeof(double) * rows * TRACE_COLS, cudaMemcpyDeviceToHost));
  return rows;
}

static int ensure_staging(omg_problem* h, int B, int shared) {
  if (B <= h->hostB && shared == h->host_shared) return 0;
  void** st[] = {(void**)&h->hx0, (void**)&h->hp, (void**)&h->hlb, (void**)&h->hub, (void**)&h->hlam0,
                 (void**)&h->hx, (void**)&h->hlam, (void**)&h->hf, (void**)&h->hst, (void**)&h->hit};
  for (void** p : st) if (*p) { cudaFree(*p); *p = nullptr; }
  const size_t n = h->T.n, m = h->T.m, np_ = h->T.n_par, b = B;
  CK(cudaMalloc(&h->hx0, b * n * 8)); CK(cudaMalloc(&h->hp, b * (np_ ? np_ : 1) * 8));
  CK(cudaMalloc(&h->hlb, (shared ? 1 : b) * m * 8)); CK(cudaMalloc(&h->hub, (shared ? 1 : b) * m * 8));
  CK(cudaMalloc(&h->hlam0, b * m * 8));
  CK(cudaMalloc(&h->hx, b * n * 8)); CK(cudaMalloc(&h->hlam, b * m * 8)); CK(cudaMalloc(&h->hf, b * 8));
  CK(cudaMalloc(&h->hst, b * 4)); CK(cudaMalloc(&h->hit, b * 4));
  h->hostB = B; h->host_shared = shared;
  return 0;
}

int omg_solve_batch_host(omg_problem* h, int32_t B, const double* x0, const double* p,
                         const double* lbg, const double* ubg, int32_t bounds_shared,
                         const double* lam_g0, double* x, double* lam_g, double* f,
                         int32_t* status, int32_t* iters) {
  if (!h) { set_err("null handle"); return -1; }
  if (B <= 0) return 0;
  CK(cudaSetDevice(h->device));
  if (ensure_staging(h, B, bounds_shared ? 1 : 0)) return -1;
  const size_t n = h->T.n, m = h->T.m, np_ = h->T.n_par, b = B;
  CK(cudaMemcpyAsync(h->hx0, x0, b * n * 8, cudaMemcpyHostToDevice, 0));
  CK(cudaMemcpyAsync(h->hp, p, b * np_ * 8, cudaMemcpyHostToDevice, 0));
  CK(cudaMemcpyAsync(h->hlb, lbg, (bounds_shared ? 1 : b) * m * 8, cudaMemcpyHostToDevice, 0));
  CK(cudaMemcpyAsync(h->hub, ubg, (bounds_shared ? 1 : b) * m * 8, cudaMemcpyHostToDevice, 0));
  if (lam_g0) CK(cudaMemcpyAsync(h->hlam0, lam_g0, b * m * 8, cudaMemcpyHostToDevice, 0));
  if (omg_solve_batch(h, B, h->hx0, h->hp, h->hlb, h->hub, bounds_shared, lam_g0 ? h->hlam0 : nullptr,
                      h->hx, h->hlam, h->hf, h->hst, h->hit, nullptr)) return -1;
  CK(cudaMemcpyAsync(x, h->hx, b * n * 8, cudaMemcpyDeviceToHost, 0));
  CK(cudaMemcpyAsync(lam_g, h->hlam, b * m * 8, cudaMemcpyDeviceToHost, 0));
  CK(cudaMemcpyAsync(f, h->hf, b * 8, cudaMemcpyDeviceToHost, 0));
  CK(cudaMemcpyAsync(status, h->hst, b * 4, cudaMemcpyDeviceToHost, 0));
  CK(cudaMemcpyAsync(iters, h->hit, b * 4, cudaMemcpyDeviceToHost, 0));
  CK(cudaStreamSynchronize(0));
  return 0;
}

static int ensure_feas_scratch(omg_problem* h, int grid) {
  const DevTab& T = h->T;
  const size_t n = T.n, m = T.m, n_xe = n + 1 + T.n_mid;
  const size_t stride = ((size_t)T.n_v + T.nnz_jx + 2 * m + n * n + (n + 1) * n + 2 * n + 2 * n_xe + 7) & ~(size_t)7;
  if (grid > h->fscr_ctas) {
    if (h->fscr) cudaFree(h->fscr);
    h->fscr = nullptr; h->fscr_ctas = 0;
    CK(cudaMalloc(&h->fscr, (size_t)grid * stride * sizeof(double)));
    h->fscr_ctas = grid;
  }
  h->fscr_stride = stride;
  return 0;
}

int omg_feas_batch(omg_problem* h, int32_t B, const double* x0, const double* p, const double* lbg,
                   const double* ubg, int32_t bounds_shared, int32_t max_steps, double* x, double* viol,
                   int32_t* steps, void* stream_) {
  if (!h) { set_err("null handle"); return -1; }
  if (B <= 0) return 0;
  if (!x0 || !p || !lbg || !ubg || !x || !viol || !steps) { set_err("null buffer"); return -1; }
  cudaStream_t stream = (cudaStream_t)stream_;
  CK(cudaSetDevice(h->device));
  int grid = h->n_sm * 2;
  if (grid > B) grid = B;
  if (ensure_feas_scratch(h, grid)) return -1;
  FeasArgs F;
  F.B = B; F.bounds_shared = bounds_shared; F.max_steps = max_steps;
  F.x0 = x0; F.p = p; F.lbg = lbg; F.ubg = ubg; F.x = x; F.viol = viol; F.steps = steps;
  F.scr = h->fscr; F.stride = h->fscr_stride;
  OMG_LAUNCH(omg_feas_kernel, grid, 256, 0, stream, h->T, F);
  CK(cudaGetLastError());
  return 0;
}

int omg_feas_batch_host(omg_problem* h, int32_t B, const double* x0, const double* p, const double* lbg,
                        const double* ubg, int32_t bounds_shared, int32_t max_steps, double* x, double* viol,
                        int32_t* steps) {
  if (!h) { set_err("null handle"); return -1; }
  if (B <= 0) return 0;
  CK(cudaSetDevice(h->device));
  if (ensure_staging(h, B, bounds_shared ? 1 : 0)) return -1;
  const size_t n = h->T.n, m = h->T.m, np_ = h->T.n_par, b = B;
  CK(cudaMemcpyAsync(h->hx0, x0, b * n * 8, cudaMemcpyHostToDevice, 0));
  CK(cudaMemcpyAsync(h->hp, p, b * np_ * 8, cudaMemcpyHostToDevice, 0));
  CK(cudaMemcpyAsync(h->hlb, lbg, (bounds_shared ? 1 : b) * m * 8, cudaMemcpyHostToDevice, 0));
  CK(cudaMemcpyAsync(h->hub, ubg, (bounds_shared ? 1 : b) * m * 8, cudaMemcpyHostToDevice, 0));
  if (omg_feas_batch(h, B, h->hx0, h->hp, h->hlb, h->hub, bounds_shared, max_steps, h->hx, h->hf, h->hit, nullptr)) return -1;
  CK(cudaMemcpyAsync(x, h->hx, b * n * 8, cudaMemcpyDeviceToHost, 0));
  CK(cudaMemcpyAsync(viol, h->hf, b * 8, cudaMemcpyDeviceToHost, 0));
  CK(cudaMemcpyAsync(steps, h->hit, b * 4, cudaMemcpyDeviceToHost, 0));
  CK(cudaStreamSynchronize(0));
  return 0;
}

static int desc_upload(DescCache& c, int device, const std::vector<int>& iv, const double* dv, size_t nd,
                       cudaStream_t stream) {
  if (c.device != device || iv.size() > c.cap_i || nd > c.cap_d) {   // (re)allocate: first call / growth only
    if (c.d_i) cudaFree(c.d_i);
    if (c.d_d) cudaFree(c.d_d);
    c.d_i = nullptr; c.d_d = nullptr; c.device = -1;
    c.cap_i = std::max(iv.size(), (size_t)64) * 2; c.cap_d = std::max(nd, (size_t)64) * 2;
    CK(cudaMalloc(&c.d_i, sizeof(int) * c.cap_i));
    CK(cudaMalloc(&c.d_d, sizeof(double) * c.cap_d));
    c.device = device;
  }
  // pageable sources: the runtime stages them before returning, the caller's arrays are free again
  CK(cudaMemcpyAsync(c.d_i, iv.data(), sizeof(int) * iv.size(), cudaMemcpyHostToDevice, stream));
  CK(cudaMemcpyAsync(c.d_d, dv, sizeof(double) * nd, cudaMemcpyHostToDevice, stream));
  return 0;
}

// Blocks of omg_shift_batch / omg_sample_batch (nsamp: NULL for the shift) and the x row both
// kernels hold in shared memory: false with a message naming `fn` when a block is empty or outside
// x, when the matrices or outputs (*n_mat, *n_out entries) outgrow the kernels' int offsets, or when
// the x row exceeds the shared memory of a block.  Above 48 KB the kernel `kfn` is opted in.
static bool fixed_desc(const std::string& fn, int32_t n, int32_t n_blocks, const int32_t* offs, const int32_t* lens,
                       const int32_t* ncols, const int32_t* nsamp, const void* kfn, int64_t* n_mat, int64_t* n_out) {
  *n_mat = 0; *n_out = 0;
  for (int k = 0; k < n_blocks; ++k) {
    const std::string blk = fn + ": block " + std::to_string(k) + ": ";
    if (lens[k] < 1) { set_err(blk + "basis length " + std::to_string(lens[k]) + " < 1"); return false; }
    if (nsamp && nsamp[k] < 1) { set_err(blk + "nsamp " + std::to_string(nsamp[k]) + " < 1"); return false; }
    if (ncols[k] < 1 || offs[k] < 0 || (int64_t)offs[k] + (int64_t)lens[k] * ncols[k] > n) {
      set_err(blk + "columns outside x"); return false; }
    *n_mat += (int64_t)(nsamp ? nsamp[k] : lens[k]) * lens[k];
    *n_out += (int64_t)(nsamp ? nsamp[k] : lens[k]) * ncols[k];
  }
  if (*n_mat > INT32_MAX || *n_out > INT32_MAX) { set_err(fn + ": matrices or output beyond 2^31 entries"); return false; }
  const size_t smem = sizeof(double) * (size_t)std::max<int32_t>(n, 0);
  if (smem > 227 * 1024) { set_err(fn + ": x row exceeds the shared memory of a block"); return false; }
  if (smem > 48 * 1024 &&
      cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
    set_err(fn + ": cudaFuncSetAttribute failed: " + cudaGetErrorString(cudaGetLastError())); return false; }
  return true;
}

int omg_shift_batch(omg_problem* h, int32_t B, double* x, int32_t n_blocks, const int32_t* offs,
                    const int32_t* lens, const int32_t* ncols, const double* Tm, void* stream_) {
  const std::string f("omg_shift_batch");
  if (!h || !x || !offs || !lens || !ncols || !Tm) { set_err(f + ": null argument"); return -1; }
  if (n_blocks < 0) { set_err(f + ": n_blocks " + std::to_string(n_blocks) + " < 0"); return -1; }
  CK(cudaSetDevice(h->device));
  int64_t tot = 0, n_out = 0;
  if (!fixed_desc(f, h->T.n, n_blocks, offs, lens, ncols, nullptr, (const void*)omg_shift_kernel, &tot, &n_out))
    return -1;
  if (B <= 0 || n_blocks == 0) return 0;
  cudaStream_t stream = (cudaStream_t)stream_;
  std::vector<int> iv(4 * (size_t)n_blocks);
  for (int b = 0, t = 0; b < n_blocks; ++b) {
    iv[b] = offs[b]; iv[n_blocks + b] = lens[b]; iv[2 * n_blocks + b] = ncols[b]; iv[3 * n_blocks + b] = t;
    t += lens[b] * lens[b];
  }
  if (!h->shift_desc) h->shift_desc = new DescCache();
  DescCache& c = *h->shift_desc;
  if (desc_upload(c, h->device, iv, Tm, (size_t)tot, stream)) return -1;
  OMG_LAUNCH(omg_shift_kernel, B, 128, sizeof(double) * h->T.n, stream, x, B, h->T.n, n_blocks, c.d_i, c.d_i + n_blocks,
                                                               c.d_i + 2 * n_blocks, c.d_i + 3 * n_blocks, c.d_d);
  CK(cudaGetLastError());
  return 0;
}

int omg_sample_batch(int32_t B, int32_t n, const double* x, int32_t n_blocks, const int32_t* offs,
                     const int32_t* lens, const int32_t* ncols, const int32_t* nsamp,
                     const double* Sm, double* out, void* stream_) {
  const std::string f("omg_sample_batch");
  if (!x || !offs || !lens || !ncols || !nsamp || !Sm || !out) { set_err(f + ": null argument"); return -1; }
  if (n_blocks < 0) { set_err(f + ": n_blocks " + std::to_string(n_blocks) + " < 0"); return -1; }
  int64_t stot = 0, otot = 0;
  if (!fixed_desc(f, n, n_blocks, offs, lens, ncols, nsamp, (const void*)omg_sample_kernel, &stot, &otot)) return -1;
  if (B <= 0 || n_blocks == 0) return 0;
  cudaStream_t stream = (cudaStream_t)stream_;
  std::vector<int> iv(6 * (size_t)n_blocks);
  for (int b = 0, s = 0, o = 0; b < n_blocks; ++b) {
    iv[b] = offs[b]; iv[n_blocks + b] = lens[b]; iv[2 * n_blocks + b] = ncols[b]; iv[3 * n_blocks + b] = nsamp[b];
    iv[4 * n_blocks + b] = s; s += nsamp[b] * lens[b];
    iv[5 * n_blocks + b] = o; o += nsamp[b] * ncols[b];
  }
  int device = 0;
  CK(cudaGetDevice(&device));
  static thread_local DescCache cache;         // (no handle in this call: one descriptor per host thread)
  if (desc_upload(cache, device, iv, Sm, (size_t)stot, stream)) return -1;
  const int* d_i = cache.d_i;
  OMG_LAUNCH(omg_sample_kernel, B, 128, sizeof(double) * n, stream, x, B, n, n_blocks, d_i, d_i + n_blocks, d_i + 2 * n_blocks,
                                                           d_i + 3 * n_blocks, d_i + 4 * n_blocks, d_i + 5 * n_blocks,
                                                           cache.d_d, out, otot);
  CK(cudaGetLastError());
  return 0;
}

// Descriptors of omg_shift_free_batch / omg_eval_batch (OMG_SPL_DESC ints per block, see
// omg_shift_free_kernel); false with a message naming `fn` when a block is out of bounds.  n_der
// rows of derivative coefficients per column are counted into *n_coef.
static bool spline_desc(const std::string& fn, int32_t n, int32_t n_blocks, const int32_t* offs,
                        const int32_t* lens, const int32_t* ncols, const int32_t* degrees,
                        const double* knots, int n_der, std::vector<int>& iv, size_t* n_knots,
                        int* Lmax, int* pmax, size_t* n_coef) {
  iv.assign((size_t)OMG_SPL_DESC * n_blocks, 0);
  *n_knots = 0; *n_coef = 0; *Lmax = 1; *pmax = 0;
  for (int k = 0; k < n_blocks; ++k) {
    const int L = lens[k], p = degrees[k], nc = ncols[k], off = offs[k];
    const std::string blk = fn + ": block " + std::to_string(k) + ": ";
    if (p < 0 || p > OMG_SPL_MAX_DEGREE || L < p + 1 || L > OMG_SPL_MAX_LEN) {
      set_err(blk + "degree " + std::to_string(p) + " / basis length " + std::to_string(L) + " outside 0 <= p <= " +
              std::to_string(OMG_SPL_MAX_DEGREE) + ", p + 1 <= L <= " + std::to_string(OMG_SPL_MAX_LEN));
      return false;
    }
    if (nc < 1 || off < 0 || (int64_t)off + (int64_t)L * nc > n) { set_err(blk + "columns outside x"); return false; }
    if (n_der > p + 1) {
      set_err(blk + "n_der " + std::to_string(n_der) + " above degree + 1 = " + std::to_string(p + 1)); return false; }
    const double* kk = knots + *n_knots;
    for (int j = 0; j < L + p; ++j)
      if (!(kk[j] <= kk[j + 1])) { set_err(blk + "knots not non-decreasing"); return false; }
    int* d = iv.data() + (size_t)OMG_SPL_DESC * k;
    d[0] = off; d[1] = L; d[2] = nc; d[3] = p; d[4] = (int)*n_knots; d[5] = (int)*n_coef;
    *n_knots += L + p + 1;
    *n_coef += (size_t)nc * n_der * L;
    *Lmax = std::max(*Lmax, L); *pmax = std::max(*pmax, p);
  }
  return true;
}

int omg_shift_free_batch(omg_problem* h, int32_t B, double* x, int32_t t_index, double update_time,
                         const int32_t* active, int32_t n_blocks, const int32_t* offs, const int32_t* lens,
                         const int32_t* ncols, const int32_t* degrees, const double* knots, void* stream_) {
  const std::string f("omg_shift_free_batch");
  if (!h || !x || n_blocks < 0 || (n_blocks > 0 && (!offs || !lens || !ncols || !degrees || !knots))) {
    set_err(f + ": null argument"); return -1; }
  if (!(update_time > 0.0)) { set_err(f + ": update_time must be > 0"); return -1; }
  if (t_index < 0 || t_index >= h->T.n) {
    set_err(f + ": t_index " + std::to_string(t_index) + " outside [0, " + std::to_string(h->T.n) + ")"); return -1; }
  std::vector<int> iv;
  size_t nk = 0, nco = 0;
  int Lmax = 1, pmax = 0;
  if (!spline_desc(f, h->T.n, n_blocks, offs, lens, ncols, degrees, knots, 1, iv, &nk, &Lmax, &pmax, &nco)) return -1;
  if (B <= 0) return 0;
  const int nt = 128;
  const size_t smem = sizeof(double) * ((size_t)h->T.n + 2 * (size_t)Lmax + pmax + 1 + 2 * nt + 2 * (size_t)Lmax * Lmax);
  if (smem > 227 * 1024) { set_err(f + ": x row and bases exceed the shared memory of a block"); return -1; }
  cudaStream_t stream = (cudaStream_t)stream_;
  CK(cudaSetDevice(h->device));
  static thread_local DescCache cache;         // (one descriptor per host thread, as omg_sample_batch)
  if (desc_upload(cache, h->device, iv, knots, nk, stream)) return -1;
  if (smem > 48 * 1024)
    CK(cudaFuncSetAttribute((const void*)omg_shift_free_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  OMG_LAUNCH(omg_shift_free_kernel, B, nt, smem, stream, x, B, h->T.n, t_index, update_time, active, n_blocks,
             cache.d_i, cache.d_d, Lmax, pmax);
  CK(cudaGetLastError());
  return 0;
}

int omg_eval_batch(int32_t B, int32_t n, const double* x, int32_t n_blocks, const int32_t* offs,
                   const int32_t* lens, const int32_t* ncols, const int32_t* degrees, const double* knots,
                   int32_t n_pts, const double* tau, const double* scale, int32_t n_der, double* out,
                   void* stream_) {
  const std::string f("omg_eval_batch");
  if (!x || !tau || !scale || !out || n_blocks < 0 ||
      (n_blocks > 0 && (!offs || !lens || !ncols || !degrees || !knots))) { set_err(f + ": null argument"); return -1; }
  if (n_der < 1 || n_der > 4) { set_err(f + ": n_der " + std::to_string(n_der) + " outside 1 .. 4"); return -1; }
  if (n_pts < 1) { set_err(f + ": n_pts must be >= 1"); return -1; }
  std::vector<int> iv;
  size_t nk = 0, nco = 0;
  int Lmax = 1, pmax = 0;
  if (!spline_desc(f, n, n_blocks, offs, lens, ncols, degrees, knots, n_der, iv, &nk, &Lmax, &pmax, &nco)) return -1;
  if (nco * sizeof(double) > 48 * 1024) { set_err(f + ": derivative coefficients exceed 48 KB per instance"); return -1; }
  if (B <= 0 || n_blocks == 0) return 0;
  int n_out = 0;
  for (int k = 0; k < n_blocks; ++k) n_out += ncols[k] * n_pts * n_der;
  cudaStream_t stream = (cudaStream_t)stream_;
  int device = 0;
  CK(cudaGetDevice(&device));
  static thread_local DescCache cache;
  if (desc_upload(cache, device, iv, knots, nk, stream)) return -1;
  OMG_LAUNCH(omg_eval_kernel, B, 64, sizeof(double) * nco, stream, x, B, n, n_blocks, cache.d_i, cache.d_d, n_pts,
             tau, scale, n_der, out, n_out);
  CK(cudaGetLastError());
  return 0;
}

int omg_integrate_rk4(int32_t model, int32_t B, int32_t n_state, int32_t n_input, const double* state0,
                      const double* inputs, double sample_time, int32_t steps, double* stateT, void* stream_) {
  if (B <= 0) return 0;
  if (!state0 || !inputs || !stateT) { set_err("null buffer"); return -1; }
  if (model < 0 || model >= OMG_ODE_N_MODELS || n_state < 1 || n_state > OMG_ODE_MAX_STATE || steps < 0 ||
      !omg_ode_sizes_ok(model, n_state, n_input)) { set_err("bad vehicle model / sizes"); return -1; }
  cudaStream_t stream = (cudaStream_t)stream_;
  OMG_LAUNCH(omg_rk4_kernel, (B + 127) / 128, 128, 0, stream, omg_ode_models[model].ode, B, n_state, n_input,
             state0, inputs, sample_time, steps, stateT);
  CK(cudaGetLastError());
  return 0;
}

// omg_closed_loop_step, omg_closed_loop_step_der and omg_closed_loop_step_fleet; `fn` names the
// caller in the messages.  R holds the rows [n_der][n_samp+1][L], except row 1 when R1 is given
// (omg_closed_loop_step's separate R0 and R1).  veh_off [n_veh]: host offsets of the vehicles'
// spline blocks in x.
static int closed_loop_launch(const char* fn, int32_t model, int32_t B, int32_t n_veh, int32_t n_state,
                              int32_t n_input, int32_t n, const double* x, const int32_t* veh_off, int32_t L,
                              int32_t n_samp, int32_t n_der, const double* R,
                              const double* R1, double sample_time, int32_t lag, double time_constant, int32_t disturb, int32_t n_traj,
                              const double* filt, const double* mean, const double* stdev, uint64_t seed,
                              int32_t step, const double* plant_x, const double* plant_u, double* plant_x_next,
                              double* plant_u_next, double* pred_x, double* pred_u, double* scratch, void* stream_) {
  const std::string f(fn);
  if (model < 0 || model >= OMG_ODE_N_MODELS) { set_err(f + ": unknown vehicle model " + std::to_string(model)); return -1; }
  const bool sizes_ok = omg_ode_sizes_ok(model, n_state, n_input) && n_input <= OMG_CL_MAX_INPUT && n >= n_input * L;
  if (!sizes_ok || L < 1 || n_samp < 0) { set_err(f + ": bad state / input / spline sizes"); return -1; }
  if (n_veh < 1) { set_err(f + ": n_veh must be >= 1, got " + std::to_string(n_veh)); return -1; }
  if (!veh_off) { set_err(f + ": null argument (vehicle offsets)"); return -1; }
  for (int v = 0; v < n_veh; ++v)
    if (veh_off[v] < 0 || (int64_t)veh_off[v] + (int64_t)n_input * L > n) {
      set_err(f + ": vehicle " + std::to_string(v) + " at offset " + std::to_string(veh_off[v]) + ": its " +
              std::to_string(n_input) + " input splines of length " + std::to_string(L) + " leave x of " +
              std::to_string(n) + " variables"); return -1; }
  if (n_der < omg_ode_models[model].n_der || n_der > 4) {
    set_err(f + ": vehicle model " + std::to_string(model) + " needs " + std::to_string(omg_ode_models[model].n_der) +
            " to 4 derivative rows, got " + std::to_string(n_der)); return -1; }
  // three [n_samp+1][n_input] arrays in the default 48 KB of dynamic shared memory
  if ((int64_t)(n_samp + 1) * n_input > 2048) {
    set_err(f + ": (n_samp + 1) * n_input exceeds 2048 samples per update"); return -1; }
  if (!(sample_time > 0.0)) { set_err(f + ": sample_time must be > 0"); return -1; }
  if (lag && !(time_constant > 0.0)) { set_err(f + ": time_constant must be > 0 with the lag on"); return -1; }
  if (disturb && n_traj <= OMG_CL_PAD) {
    set_err(f + ": n_traj must exceed the filter padding of 12 samples"); return -1; }
  if (disturb && n_traj < n_samp + 1) { set_err(f + ": n_traj < n_samp + 1"); return -1; }
  if (!x || !R || !plant_x || !plant_u || !plant_x_next || !plant_u_next || !pred_x || !pred_u ||
      (disturb && (!filt || !mean || !stdev || !scratch))) { set_err(f + ": null argument"); return -1; }
  if (B <= 0) return 0;
  if ((int64_t)B * n_veh > 0x7fffffff) { set_err(f + ": B * n_veh exceeds 2^31 - 1 blocks"); return -1; }
  cudaStream_t stream = (cudaStream_t)stream_;
  // host descriptors -> device: R (the rows the model reads) | filt (11) | mean | stdev
  const size_t nr = (size_t)(n_samp + 1) * L, nR = (size_t)omg_ode_models[model].n_der * nr;
  std::vector<double> dv(nR + 11 + 2 * (size_t)n_input, 0.0);
  for (int r = 0; r < omg_ode_models[model].n_der; ++r) {
    const double* src = r == 1 && R1 ? R1 : R + r * nr;
    std::copy(src, src + nr, dv.begin() + r * nr);
  }
  if (disturb) {
    std::copy(filt, filt + 11, dv.begin() + nR);
    std::copy(mean, mean + n_input, dv.begin() + nR + 11);
    std::copy(stdev, stdev + n_input, dv.begin() + nR + 11 + n_input);
  }
  int device = 0;
  CK(cudaGetDevice(&device));
  static thread_local DescCache cache;
  if (desc_upload(cache, device, std::vector<int>(veh_off, veh_off + n_veh), dv.data(), dv.size(), stream)) return -1;
  const double* d = cache.d_d;
  const size_t smem = sizeof(double) * 3 * (size_t)(n_samp + 1) * n_input;
  OMG_LAUNCH(omg_closed_loop_kernel, B * n_veh, 32, smem, stream, model, omg_ode_models[model].ode,
             omg_ode_models[model].n_der, n_state, n_input, n, n_veh, cache.d_i, x,
             L, n_samp, d, sample_time, lag, time_constant, disturb, n_traj, d + nR, d + nR + 11,
             d + nR + 11 + n_input, seed, step, plant_x, plant_u, plant_x_next, plant_u_next, pred_x, pred_u, scratch);
  CK(cudaGetLastError());
  return 0;
}

int omg_closed_loop_step_der(int32_t model, int32_t B, int32_t n_state, int32_t n_input, int32_t n, const double* x,
                             int32_t L, int32_t n_samp, int32_t n_der, const double* R, double sample_time,
                             int32_t lag, double time_constant, int32_t disturb, int32_t n_traj, const double* filt,
                             const double* mean, const double* stdev, uint64_t seed, int32_t step,
                             const double* plant_x, const double* plant_u, double* plant_x_next,
                             double* plant_u_next, double* pred_x, double* pred_u, double* scratch, void* stream) {
  const int32_t off0 = 0;
  return closed_loop_launch("omg_closed_loop_step_der", model, B, 1, n_state, n_input, n, x, &off0, L, n_samp, n_der,
                            R, nullptr, sample_time, lag, time_constant, disturb, n_traj, filt, mean, stdev, seed, step,
                            plant_x, plant_u, plant_x_next, plant_u_next, pred_x, pred_u, scratch, stream);
}

int omg_closed_loop_step_fleet(int32_t model, int32_t B, int32_t n_veh, int32_t n_state, int32_t n_input, int32_t n,
                               const double* x, const int32_t* veh_off, int32_t L, int32_t n_samp, int32_t n_der,
                               const double* R, double sample_time, int32_t lag, double time_constant,
                               int32_t disturb, int32_t n_traj, const double* filt, const double* mean,
                               const double* stdev, uint64_t seed, int32_t step, const double* plant_x,
                               const double* plant_u, double* plant_x_next, double* plant_u_next, double* pred_x,
                               double* pred_u, double* scratch, void* stream) {
  return closed_loop_launch("omg_closed_loop_step_fleet", model, B, n_veh, n_state, n_input, n, x, veh_off, L, n_samp,
                            n_der, R, nullptr, sample_time, lag, time_constant, disturb, n_traj, filt, mean, stdev,
                            seed, step, plant_x, plant_u, plant_x_next, plant_u_next, pred_x, pred_u, scratch, stream);
}

int omg_closed_loop_step(int32_t model, int32_t B, int32_t n_state, int32_t n_input, int32_t n, const double* x,
                         int32_t L, int32_t n_samp, const double* R0, const double* R1, double sample_time,
                         int32_t lag, double time_constant, int32_t disturb, int32_t n_traj, const double* filt,
                         const double* mean, const double* stdev, uint64_t seed, int32_t step,
                         const double* plant_x, const double* plant_u, double* plant_x_next, double* plant_u_next,
                         double* pred_x, double* pred_u, double* scratch, void* stream) {
  if (model != OMG_ODE_INTEGRATOR && model != OMG_ODE_QUADROTOR3D) {
    set_err("omg_closed_loop_step: unknown vehicle model " + std::to_string(model)); return -1; }
  if (!R1) R0 = nullptr;                            // (reported as a null argument)
  const int32_t off0 = 0;
  return closed_loop_launch("omg_closed_loop_step", model, B, 1, n_state, n_input, n, x, &off0, L, n_samp, 2, R0, R1,
                            sample_time, lag, time_constant, disturb, n_traj, filt, mean, stdev, seed, step, plant_x,
                            plant_u, plant_x_next, plant_u_next, pred_x, pred_u, scratch, stream);
}

int omg_closed_loop_step_free(int32_t model, int32_t B, int32_t n_state, int32_t n_input, int32_t n, const double* x,
                              int32_t spl_offset, int32_t L, int32_t n_cols, int32_t degree, const double* knots,
                              int32_t t_index, int32_t n_der, const int32_t* n_samp, const int32_t* n_traj,
                              double sample_time, int32_t lag, double time_constant, int32_t disturb,
                              const double* filt, const double* mean, const double* stdev, uint64_t seed, int32_t step,
                              const double* plant_x, const double* plant_u, double* plant_x_next, double* plant_u_next,
                              double* pred_x, double* pred_u, double* scratch, void* stream_) {
  const std::string f("omg_closed_loop_step_free");
  if (model < 0 || model >= OMG_ODE_N_MODELS) { set_err(f + ": unknown vehicle model " + std::to_string(model)); return -1; }
  const bool sizes_ok = omg_ode_sizes_ok(model, n_state, n_input) && n_input <= OMG_CL_MAX_INPUT;
  if (!sizes_ok || B < 0) { set_err(f + ": bad state / input sizes"); return -1; }
  if (n_der < omg_ode_models[model].n_der || n_der > 4) {
    set_err(f + ": vehicle model " + std::to_string(model) + " needs " + std::to_string(omg_ode_models[model].n_der) +
            " to 4 derivative rows, got " + std::to_string(n_der)); return -1; }
  if (!x || !knots || !n_samp || !plant_x || !plant_u || !plant_x_next || !plant_u_next || !pred_x || !pred_u ||
      (disturb && (!n_traj || !filt || !mean || !stdev || !scratch))) { set_err(f + ": null argument"); return -1; }
  std::vector<int> iv;
  size_t nk = 0, nco = 0;
  int Lmax = 1, pmax = 0;
  if (!spline_desc(f, n, 1, &spl_offset, &L, &n_cols, &degree, knots, n_der, iv, &nk, &Lmax, &pmax, &nco)) return -1;
  if (n_cols < n_input) {
    set_err(f + ": the spline block has " + std::to_string(n_cols) + " columns, the model reads " +
            std::to_string(n_input)); return -1; }
  if (t_index < 0 || t_index >= n) {
    set_err(f + ": t_index " + std::to_string(t_index) + " outside [0, " + std::to_string(n) + ")"); return -1; }
  if (!(sample_time > 0.0)) { set_err(f + ": sample_time must be > 0"); return -1; }
  if (lag && !(time_constant > 0.0)) { set_err(f + ": time_constant must be > 0 with the lag on"); return -1; }
  int ns_max = 0, nt_max = 0;
  for (int b = 0; b < B; ++b) {
    const std::string inst = f + ": instance " + std::to_string(b) + ": ";
    if (n_samp[b] < 0) { set_err(inst + "n_samp < 0"); return -1; }
    ns_max = std::max(ns_max, (int)n_samp[b]);
    if (!disturb) continue;
    const int nt = n_traj[b];
    if (nt < 0 || (nt > 0 && nt <= OMG_CL_PAD)) {
      set_err(inst + "n_traj must be 0 or exceed the filter padding of 12 samples"); return -1; }
    if (nt > 0 && nt < n_samp[b] + 1) { set_err(inst + "n_traj < n_samp + 1"); return -1; }
    nt_max = std::max(nt_max, nt);
  }
  // three [n_samp+1][n_input] arrays for the largest update
  if ((int64_t)(ns_max + 1) * n_input > 2048) {
    set_err(f + ": (max n_samp + 1) * n_input exceeds 2048 samples per update"); return -1; }
  if (B == 0 || ns_max == 0) return 0;
  cudaStream_t stream = (cudaStream_t)stream_;
  // host descriptors -> device: ints {desc (4) | n_samp [B] | n_traj [B]}, doubles {knots | filt (11) | mean | stdev}
  std::vector<int> di(4 + 2 * (size_t)B, 0);
  std::copy(iv.begin(), iv.begin() + 4, di.begin());
  std::copy(n_samp, n_samp + B, di.begin() + 4);
  if (disturb) std::copy(n_traj, n_traj + B, di.begin() + 4 + B);
  std::vector<double> dv(nk + 11 + 2 * (size_t)n_input, 0.0);
  std::copy(knots, knots + nk, dv.begin());
  if (disturb) {
    std::copy(filt, filt + 11, dv.begin() + nk);
    std::copy(mean, mean + n_input, dv.begin() + nk + 11);
    std::copy(stdev, stdev + n_input, dv.begin() + nk + 11 + n_input);
  }
  int device = 0;
  CK(cudaGetDevice(&device));
  static thread_local DescCache cache;
  if (desc_upload(cache, device, di, dv.data(), dv.size(), stream)) return -1;
  const int* d_i = cache.d_i;
  const double* d = cache.d_d;
  const int ts_max = ns_max + 1;
  const size_t smem = sizeof(double) * (3 * (size_t)ts_max * n_input + (size_t)n_input * n_der * L);
  if (smem > 48 * 1024)
    CK(cudaFuncSetAttribute((const void*)omg_closed_loop_free_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                            (int)smem));
  OMG_LAUNCH(omg_closed_loop_free_kernel, B, 32, smem, stream, model, omg_ode_models[model].ode, n_der, n_state,
             n_input, n, x, d_i, d, t_index, d_i + 4, d_i + 4 + B, ts_max, sample_time, lag, time_constant, disturb,
             d + nk, d + nk + 11, d + nk + 11 + n_input, seed, step, plant_x, plant_u, plant_x_next, plant_u_next,
             pred_x, pred_u, scratch, (size_t)nt_max + 2 * OMG_CL_PAD);
  CK(cudaGetLastError());
  return 0;
}

int omg_admm_zl_update(int32_t n_agents, int32_t nsh, int32_t n_nghb, int32_t L,
                       const double* PzT, const double* c, const double* Tf, const double* Tb,
                       double rho, const double* x_i, const double* x_j, double* z_i, double* z_ij,
                       double* l_i, double* l_ij, double* res, void* stream_) {
  if (n_agents <= 0) return 0;
  if (!PzT || !c || !Tf || !Tb || !x_i || !x_j || !z_i || !z_ij || !l_i || !l_ij || !res) { set_err("null buffer"); return -1; }
  const int nz = nsh * (1 + n_nghb);
  int nt = 32; while (nt < nz) nt <<= 1;
  if (nt > 1024 || nsh % L != 0) { set_err("unsupported consensus block size"); return -1; }
  const size_t smem = sizeof(double) * (5 * (size_t)nz + 64);
  OMG_LAUNCH(omg_admm_zl_kernel, n_agents, nt, smem, (cudaStream_t)stream_, nsh, n_nghb, L, PzT, c, Tf, Tb, rho,
                                                                   x_i, x_j, z_i, z_ij, l_i, l_ij, res);
  CK(cudaGetLastError());
  return 0;
}

// ---- multi-GPU ADMM exchange (NCCL bound at run time) -----------------------------------------
struct omg_comm {
  int n_ranks = 1, rank = 0, device = 0;
  void* nccl = nullptr;                 // ncclComm_t
  double* gx = nullptr; double* gz = nullptr; double* gl = nullptr; size_t cap_x = 0, cap_z = 0;
};

}  // extern "C" (reopened below)

#ifndef OMG_CPU_EMU
#include <dlfcn.h>
#endif
struct OmgNcclId { char internal[128]; };      // layout of ncclUniqueId
namespace {
struct NcclApi {
  bool ok = false;
  int (*GetUniqueId)(void*) = nullptr;
  int (*CommInitRank)(void**, int, OmgNcclId /* ncclUniqueId by value */, int) = nullptr;
  int (*CommDestroy)(void*) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
  int (*AllReduce)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
};
NcclApi g_nccl;
const int kNcclFloat64 = 8, kNcclSum = 0;

bool nccl_bind() {
#ifdef OMG_CPU_EMU
  return false;
#else
  if (g_nccl.ok) return true;
  void* lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD | RTLD_GLOBAL);   // the host process' copy, if any
  if (!lib) lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!lib) lib = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (!lib) { set_err("NCCL not found (dlopen libnccl.so.2)"); return false; }
  *(void**)(&g_nccl.GetUniqueId) = dlsym(lib, "ncclGetUniqueId");
  *(void**)(&g_nccl.CommInitRank) = dlsym(lib, "ncclCommInitRank");
  *(void**)(&g_nccl.CommDestroy) = dlsym(lib, "ncclCommDestroy");
  *(void**)(&g_nccl.AllGather) = dlsym(lib, "ncclAllGather");
  *(void**)(&g_nccl.AllReduce) = dlsym(lib, "ncclAllReduce");
  *(void**)(&g_nccl.GetErrorString) = dlsym(lib, "ncclGetErrorString");
  g_nccl.ok = g_nccl.GetUniqueId && g_nccl.CommInitRank && g_nccl.CommDestroy && g_nccl.AllGather &&
              g_nccl.AllReduce && g_nccl.GetErrorString;
  if (!g_nccl.ok) set_err("libnccl lacks a required symbol");
  return g_nccl.ok;
#endif
}
#define NK(call) do { int r_ = (call); if (r_ != 0) { set_err(std::string(#call) + ": " + g_nccl.GetErrorString(r_)); return -1; } } while (0)

// dst[i][k][:] = src[idx_a[i][k]] [ idx_b ? idx_b[i][k] : - ] [:]  (rows of `len` doubles)
__global__ void omg_gather_rows_kernel(int n_rows, int len, int stride_a, const int* __restrict__ ia,
                                       const int* __restrict__ ib, const double* __restrict__ src,
                                       double* __restrict__ dst) {
  const int r = blockIdx.x;
  if (r >= n_rows) return;
  const size_t base = (size_t)ia[r] * stride_a + (ib ? (size_t)ib[r] * len : 0);
  for (int q = threadIdx.x; q < len; q += blockDim.x) dst[(size_t)r * len + q] = src[base + q];
}
__global__ void omg_colsum3_kernel(int n, const double* __restrict__ res, double* __restrict__ out) {
  double a = 0.0;
  for (int i = 0; i < n; ++i) a += res[(size_t)i * 3 + threadIdx.x];   // fixed order: deterministic
  out[threadIdx.x] = a;
}
}  // namespace

extern "C" {

int omg_comm_unique_id(void* id128) {
  if (!id128) { set_err("null buffer"); return -1; }
  if (!nccl_bind()) return -1;
  NK(g_nccl.GetUniqueId(id128));
  return 0;
}

omg_comm* omg_comm_create(const void* id128, int32_t n_ranks, int32_t rank, int32_t device) {
  if (n_ranks < 1 || rank < 0 || rank >= n_ranks) { set_err("bad rank / n_ranks"); return nullptr; }
  if (cudaSetDevice(device) != cudaSuccess) { set_err("cudaSetDevice failed"); return nullptr; }
  omg_comm* c = new omg_comm();
  c->n_ranks = n_ranks; c->rank = rank; c->device = device;
  if (n_ranks > 1) {
    if (!id128 || !nccl_bind()) { if (!id128) set_err("null unique id"); delete c; return nullptr; }
    OmgNcclId id; memcpy(&id, id128, sizeof id);
    const int r = g_nccl.CommInitRank(&c->nccl, n_ranks, id, rank);
    if (r != 0) { set_err(std::string("ncclCommInitRank: ") + g_nccl.GetErrorString(r)); delete c; return nullptr; }
  }
  return c;
}

void omg_comm_destroy(omg_comm* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  if (c->nccl && g_nccl.ok) g_nccl.CommDestroy(c->nccl);
  if (c->gx) cudaFree(c->gx);
  if (c->gz) cudaFree(c->gz);
  if (c->gl) cudaFree(c->gl);
  delete c;
}

static int comm_reserve(omg_comm* c, size_t nx, size_t nz) {
  if (nx > c->cap_x) { if (c->gx) cudaFree(c->gx); c->gx = nullptr; CK(cudaMalloc(&c->gx, nx * 8)); c->cap_x = nx; }
  if (nz > c->cap_z) {
    if (c->gz) cudaFree(c->gz); if (c->gl) cudaFree(c->gl); c->gz = c->gl = nullptr;
    CK(cudaMalloc(&c->gz, nz * 8)); CK(cudaMalloc(&c->gl, nz * 8)); c->cap_z = nz;
  }
  return 0;
}

int omg_admm_exchange_x(omg_comm* c, int32_t n_local, int32_t nsh, int32_t n_nghb, const int32_t* nghb,
                        const double* x_i, double* x_j, void* stream_) {
  if (!c || !nghb || !x_i || !x_j) { set_err("null argument"); return -1; }
  if (n_local <= 0) return 0;
  cudaStream_t stream = (cudaStream_t)stream_;
  CK(cudaSetDevice(c->device));
  const double* all = x_i;
  if (c->n_ranks > 1) {
    if (comm_reserve(c, (size_t)c->n_ranks * n_local * nsh, 0)) return -1;
    NK(g_nccl.AllGather(x_i, c->gx, (size_t)n_local * nsh, kNcclFloat64, c->nccl, stream));
    all = c->gx;
  }
  OMG_LAUNCH(omg_gather_rows_kernel, n_local * n_nghb, 32, 0, stream, n_local * n_nghb, nsh, nsh, nghb,
             (const int*)nullptr, all, x_j);
  CK(cudaGetLastError());
  return 0;
}

int omg_admm_zl_update_dist(omg_comm* c, int32_t n_local, int32_t nsh, int32_t n_nghb, int32_t L,
                            const double* PzT, const double* cvec, const double* Tf, const double* Tb,
                            double rho, const double* x_i, const double* x_j, double* z_i, double* z_ij,
                            double* l_i, double* l_ij, double* res, const int32_t* nghb, const int32_t* back,
                            double* z_ji, double* l_ji, double* res_total, void* stream_) {
  if (!c || !nghb || !back || !z_ji || !l_ji || !res_total) { set_err("null argument"); return -1; }
  if (n_local <= 0) return 0;
  cudaStream_t stream = (cudaStream_t)stream_;
  CK(cudaSetDevice(c->device));
  if (omg_admm_zl_update(n_local, nsh, n_nghb, L, PzT, cvec, Tf, Tb, rho, x_i, x_j, z_i, z_ij, l_i, l_ij,
                         res, stream_)) return -1;
  OMG_LAUNCH(omg_colsum3_kernel, 1, 3, 0, stream, n_local, res, res_total);
  CK(cudaGetLastError());
  const double* allz = z_ij; const double* alll = l_ij;
  if (c->n_ranks > 1) {
    const size_t cnt = (size_t)n_local * n_nghb * nsh;
    if (comm_reserve(c, 0, (size_t)c->n_ranks * cnt)) return -1;
    NK(g_nccl.AllReduce(res_total, res_total, 3, kNcclFloat64, kNcclSum, c->nccl, stream));
    NK(g_nccl.AllGather(z_ij, c->gz, cnt, kNcclFloat64, c->nccl, stream));
    NK(g_nccl.AllGather(l_ij, c->gl, cnt, kNcclFloat64, c->nccl, stream));
    allz = c->gz; alll = c->gl;
  }
  OMG_LAUNCH(omg_gather_rows_kernel, n_local * n_nghb, 32, 0, stream, n_local * n_nghb, nsh, n_nghb * nsh, nghb, back, allz, z_ji);
  OMG_LAUNCH(omg_gather_rows_kernel, n_local * n_nghb, 32, 0, stream, n_local * n_nghb, nsh, n_nghb * nsh, nghb, back, alll, l_ji);
  CK(cudaGetLastError());
  return 0;
}

}  // extern "C"

// ===========================================================================
// Device-resident receding-horizon update (include/omg_b200.h: omg_mpc_*), the batched
// Point2Point::update() of the reference's export (Point2Point.cpp:119-231) for one Holonomic /
// Holonomic3D vehicle with a fixed horizon.  Two kernels around omg_solve_batch, one instance
// per block: prepare (cold start or knot shift, prediction, parameter row) and commit (accept or
// keep, trajectory samples, the next prediction).
// ===========================================================================
struct MpcDev {
  int B, n, n_par, nd, spl_off, L, p, traj_len, n_samp, mode, n_obs, n_shift;
  int p_state0, p_input0, p_poseT, p_t, p_T;
  double horizon, knot_time, update_time, sample_time;
  const double* knots;      // [L + p + 1]
  const int* obs_kind;      // [n_obs]
  const int* obs_off;       // [n_obs][4]
  const int* shift_desc;    // [n_shift][4]: offset in x, len, columns, offset of its T in shift_T
  const double* shift_T;
  const double* x_tpl;      // [n]
  const double* p_tpl;      // [n_par]
  double* X;                // [B][n] the warm start of the next update (last accepted solution)
  double* X0;               // [B][n] the warm start handed to the solve
  double* Xn;               // [B][n] the solve's result
  double* P;                // [B][n_par]
  double* t;                // [B] instance time
  double* t_prev;           // [B]
  double* pred_x;           // [B][nd] ideal prediction: state at t_rel + update_time
  double* pred_u;           // [B][nd] and input
  double* U;                // [B][n_samp + 1][nd] integrate: planned inputs from t_rel
  int* rec;                 // [B] cold start requested by omg_mpc_recover
  // free motion time (omg_mpc_create_freet)
  int t_index, n_blocks, Lmax, pmax;
  double stop_tol;
  const int* blk_desc;      // [n_blocks][OMG_SPL_DESC] the shifted spline blocks (spline_desc)
  const double* blk_knots;
  double* Tm;               // [B] T of the last accepted plan
  int* phase;               // [B] OMG_MPC_COLD / _ACCEPTED / _FAILED: what the last update left
  int* stop;                // [B] stopped (not solved until omg_mpc_recover)
  int* ns;                  // [B] integrate: the samples of U the next prediction spans
  int* rows;                // [B] the rows solved by this update, ascending
  int* n_rows;              // [1]
  // obstacle shapes and avoidance (omg_mpc_attach_obstacles); shapes == nullptr: not attached
  int m, n_shape;           // g rows; doubles of one instance's shape record
  const int* obs_geo;       // [n_obs][6]: chk_off, chk_len, rad_off, rad_len, row_off, row_len
  double* shapes;           // [B][n_shape] per obstacle its checkpoints, then its radii
  double* lbg;              // [B][m] each instance's bounds
  double* ubg;              // [B][m]
};

enum { OMG_MPC_COLD = 0, OMG_MPC_ACCEPTED = 1, OMG_MPC_FAILED = 2 };

// numpy.round(x, 6)
__device__ __forceinline__ double omg_round6(double x) { return rint(x * 1e6) / 1e6; }

// The obstacles of instance b into its parameter row pb, after the template copy (one thread): their
// x, v, a (and theta) from obs[b] and, with obstacles attached, their stored checkpoints and radii.
__device__ void omg_mpc_write_obstacles(const MpcDev& M, int b, const double* __restrict__ obs, double* pb) {
  const int nd = M.nd, rl = 3 * nd + 1;
  for (int k = 0; k < M.n_obs; ++k) {
    const double* o = obs + ((size_t)b * M.n_obs + k) * rl;
    const int* off = M.obs_off + 4 * k;
    for (int c = 0; c < nd; ++c) {
      pb[off[0] + c] = o[c];
      pb[off[1] + c] = o[nd + c];
      pb[off[2] + c] = o[2 * nd + c];
    }
    if (M.obs_kind[k]) pb[off[3]] = o[3 * nd];
  }
  if (!M.shapes) return;
  const double* s = M.shapes + (size_t)b * M.n_shape;
  for (int k = 0; k < M.n_obs; ++k) {
    const int* g = M.obs_geo + 6 * k;
    for (int i = 0; i < g[1]; ++i) pb[g[0] + i] = *s++;
    for (int i = 0; i < g[3]; ++i) pb[g[2] + i] = *s++;
  }
}

// Shared memory: source x row [n] | warm start [n].
__global__ void omg_mpc_prepare_kernel(const MpcDev M, const double* __restrict__ state0,
                                       const double* __restrict__ stateT, const double* __restrict__ obs) {
  OMG_DYN_SHARED(xs);
  const int b = blockIdx.x, t = threadIdx.x, nt = blockDim.x, n = M.n, nd = M.nd, L = M.L;
  if (b >= M.B) return;
  double* ws = xs + n;
  const double tb = M.t[b], kt = M.knot_time;
  const bool cold = fabs(tb) <= 1e-6 || M.rec[b] != 0;
  const bool cross = !cold && (long long)omg_round6(M.t_prev[b] / kt) < (long long)omg_round6(tb / kt);
  const double* src = cold ? M.x_tpl : M.X + (size_t)b * n;
  for (int i = t; i < n; i += nt) xs[i] = ws[i] = src[i];
  __syncthreads();
  if (cold) {                         // getInitSplineValue: linspace(state0, stateT, L) per column
    for (int e = t; e < nd * L; e += nt) {
      const int c = e / L, i = e - c * L;
      ws[M.spl_off + e] = omg_linspace(state0[(size_t)b * nd + c], stateT[(size_t)b * nd + c], L, i);
    }
  } else if (cross) {                 // transformSplines
    for (int k = 0; k < M.n_shift; ++k) {
      const int* d = M.shift_desc + 4 * k;
      omg_shift_block(M.shift_T + d[3], xs, ws, d[0], d[1], d[2]);
    }
  }
  __syncthreads();
  double* x0 = M.X0 + (size_t)b * n;
  double* pb = M.P + (size_t)b * M.n_par;
  for (int i = t; i < n; i += nt) x0[i] = ws[i];
  for (int i = t; i < M.n_par; i += nt) pb[i] = M.p_tpl[i];
  __syncthreads();                    // (the template row is in place; every thread has read rec[b])
  if (t != 0) return;
  double s0[OMG_ODE_MAX_STATE], u0[OMG_CL_MAX_INPUT];
  const double* st0 = state0 + (size_t)b * nd;
  if (cold) {                         // Holonomic::setInitialConditions
    for (int c = 0; c < nd; ++c) { s0[c] = st0[c]; u0[c] = 0.0; }
  } else if (M.mode == OMG_MPC_PREDICT_IDEAL) {
    for (int c = 0; c < nd; ++c) { s0[c] = M.pred_x[(size_t)b * nd + c]; u0[c] = M.pred_u[(size_t)b * nd + c]; }
  } else {                            // RK4 from the measured state over the planned inputs
    const double* Ub = M.U + (size_t)b * (M.n_samp + 1) * nd;
    for (int c = 0; c < nd; ++c) s0[c] = st0[c];
    double st[OMG_ODE_MAX_STATE], k1[OMG_ODE_MAX_STATE], k2[OMG_ODE_MAX_STATE], k3[OMG_ODE_MAX_STATE],
           k4[OMG_ODE_MAX_STATE], um[OMG_CL_MAX_INPUT];
    omg_rk4_interp(OMG_ODE_INTEGRATOR, nd, nd, M.n_samp, M.sample_time, Ub, s0, st, k1, k2, k3, k4, um);
    for (int c = 0; c < nd; ++c) u0[c] = Ub[(size_t)M.n_samp * nd + c];
  }
  for (int c = 0; c < nd; ++c) {
    pb[M.p_state0 + c] = s0[c];
    pb[M.p_input0 + c] = u0[c];
    pb[M.p_poseT + c] = stateT[(size_t)b * nd + c];
  }
  pb[M.p_t] = fmod(omg_round6(tb), kt);
  pb[M.p_T] = M.horizon;
  omg_mpc_write_obstacles(M, b, obs, pb);
  M.rec[b] = 0;
}

// Shared memory: the derivative coefficients (value and first derivative) of the vehicle's columns
// [nd][2][L] (omg_spl_der_coef).  Sample j < traj_len is the output row j; the samples after them
// are the next prediction's: one point at t_rel + update_time (ideal) or n_samp + 1 points at
// t_rel + s * sample_time (integrate).
__global__ void omg_mpc_commit_kernel(const MpcDev M, const int* __restrict__ status, double* __restrict__ state_traj,
                                      double* __restrict__ input_traj) {
  OMG_DYN_SHARED(cd);
  const int b = blockIdx.x, t = threadIdx.x, nt = blockDim.x, n = M.n, nd = M.nd, L = M.L, p = M.p;
  if (b >= M.B) return;
  const bool ok = status[b] == 0;
  const double tb = M.t[b];
  const double* src = (ok ? M.Xn : M.X0) + (size_t)b * n;
  double* xb = M.X + (size_t)b * n;
  for (int i = t; i < n; i += nt) xb[i] = src[i];
  if (!ok) {                          // keep the warm start and the time; do not shift again
    if (t == 0) M.t_prev[b] = tb;
    return;
  }
  for (int c = t; c < nd; c += nt) omg_spl_der_coef(M.knots, p, L, 2, src + M.spl_off + c * L, cd + (size_t)c * 2 * L);
  __syncthreads();
  const double t_rel = fmod(omg_round6(tb), M.knot_time), T = M.horizon;
  const bool ideal = M.mode == OMG_MPC_PREDICT_IDEAL;
  const int tl = M.traj_len, n_pts = tl + (ideal ? 1 : M.n_samp + 1);
  for (int j = t; j < n_pts; j += nt) {
    const double tau = j < tl ? (t_rel + (double)j * M.sample_time) / T
                       : ideal ? (t_rel + M.update_time) / T : (t_rel + (double)(j - tl) * M.sample_time) / T;
    double w[OMG_SPL_MAX_LEN + OMG_SPL_MAX_DEGREE], v[2][OMG_CL_MAX_INPUT];
    for (int d = 0; d < 2; ++d) {
      omg_cox_de_boor(M.knots + d, p - d, tau, 0, L - d, w);
      for (int c = 0; c < nd; ++c) {
        const double* q = cd + ((size_t)c * 2 + d) * L;
        double acc = 0.0;
        for (int i = 0; i < L - d; ++i) acc += w[i] * q[i];
        v[d][c] = d ? acc / T : acc;
      }
    }
    double *xo, *uo;
    if (j < tl) {
      xo = state_traj + ((size_t)b * tl + j) * nd;
      uo = input_traj + ((size_t)b * tl + j) * nd;
    } else if (ideal) {
      xo = M.pred_x + (size_t)b * nd;
      uo = M.pred_u + (size_t)b * nd;
    } else {
      xo = nullptr;
      uo = M.U + ((size_t)b * (M.n_samp + 1) + (j - tl)) * nd;
    }
    for (int c = 0; c < nd; ++c) {
      if (xo) xo[c] = v[0][c];
      uo[c] = v[1][c];
    }
  }
  __syncthreads();                    // (every thread has read t_b)
  if (t == 0) {
    M.t_prev[b] = tb;
    M.t[b] = omg_round6(tb + M.update_time);
  }
}

// Free motion time, shared memory: source x row [n] | warm start [n] | omg_shift_free_row's scratch.
// Cold start: the template with linspace(state0, stateT) in the vehicle's columns.  After an accepted
// solve: the prediction the commit stored (ideal) or RK4 from state0 over the stored inputs
// (integrate), then the stop test on the accepted plan's T and that prediction; a running instance
// is shifted from its plan's own T.  After a failed solve: the same warm start and prediction.  A
// stopped instance writes nothing.
__global__ void omg_mpc_prepare_free_kernel(const MpcDev M, const double* __restrict__ state0,
                                            const double* __restrict__ stateT, const double* __restrict__ obs) {
  OMG_DYN_SHARED(xs);
  __shared__ int stop_s;
  __shared__ double s0[OMG_ODE_MAX_STATE], u0[OMG_CL_MAX_INPUT];
  const int b = blockIdx.x, t = threadIdx.x, nt = blockDim.x, n = M.n, nd = M.nd, L = M.L;
  if (b >= M.B) return;
  double* ws = xs + n;
  const bool cold = M.rec[b] != 0 || M.phase[b] == OMG_MPC_COLD;
  const bool accepted = !cold && M.phase[b] == OMG_MPC_ACCEPTED;
  if (!cold && M.stop[b]) return;
  const double* st0 = state0 + (size_t)b * nd;
  const double* stT = stateT + (size_t)b * nd;
  if (t == 0) {
    if (cold) {                       // Holonomic::setInitialConditions
      for (int c = 0; c < nd; ++c) { s0[c] = st0[c]; u0[c] = 0.0; }
    } else if (M.mode == OMG_MPC_PREDICT_IDEAL) {
      for (int c = 0; c < nd; ++c) { s0[c] = M.pred_x[(size_t)b * nd + c]; u0[c] = M.pred_u[(size_t)b * nd + c]; }
    } else {                          // RK4 from the measured state over the planned inputs
      const double* Ub = M.U + (size_t)b * (M.n_samp + 1) * nd;
      const int ns = M.ns[b];
      double y[OMG_ODE_MAX_STATE], st[OMG_ODE_MAX_STATE], k1[OMG_ODE_MAX_STATE], k2[OMG_ODE_MAX_STATE],
             k3[OMG_ODE_MAX_STATE], k4[OMG_ODE_MAX_STATE], um[OMG_CL_MAX_INPUT];
      for (int c = 0; c < nd; ++c) y[c] = st0[c];
      omg_rk4_interp(OMG_ODE_INTEGRATOR, nd, nd, ns, M.sample_time, Ub, y, st, k1, k2, k3, k4, um);
      for (int c = 0; c < nd; ++c) { s0[c] = y[c]; u0[c] = Ub[(size_t)ns * nd + c]; }
    }
    int stop = 0;
    if (accepted) {                   // check_terminal_conditions (BatchMPC._at_goal), or T < update_time
      double e2 = 0.0, u2 = 0.0;
      for (int c = 0; c < nd; ++c) {
        const double e = s0[c] - stT[c];
        e2 = __dadd_rn(e2, __dmul_rn(e, e));
        u2 = __dadd_rn(u2, __dmul_rn(u0[c], u0[c]));
      }
      stop = M.Tm[b] < M.update_time || (sqrt(e2) <= M.stop_tol && sqrt(u2) <= M.stop_tol);
    }
    stop_s = stop;
  }
  __syncthreads();                    // (every thread has read rec[b], phase[b] and stop[b])
  if (t == 0) { M.stop[b] = stop_s; M.rec[b] = 0; }
  if (stop_s) return;
  const double* src = cold ? M.x_tpl : M.X + (size_t)b * n;
  for (int i = t; i < n; i += nt) xs[i] = ws[i] = src[i];
  __syncthreads();
  if (cold) {                         // getInitSplineValue: linspace(state0, stateT, L) per column
    for (int e = t; e < nd * L; e += nt) {
      const int c = e / L, i = e - c * L;
      ws[M.spl_off + e] = omg_linspace(st0[c], stT[c], L, i);
    }
  } else if (accepted) {              // FreeTPoint2point.init_step from the plan's own T
    double target;
    const double tau = omg_free_shift_tau(xs[M.t_index], M.update_time, &target);
    if (tau > 0.0 && tau < 1.0) {
      omg_shift_free_row(xs, ws, tau, M.n_blocks, M.blk_desc, M.blk_knots, M.Lmax, M.pmax, ws + n);
      __syncthreads();
      if (t == 0) ws[M.t_index] = target;
    }
  }
  __syncthreads();
  double* x0 = M.X0 + (size_t)b * n;
  double* pb = M.P + (size_t)b * M.n_par;
  for (int i = t; i < n; i += nt) x0[i] = ws[i];
  for (int i = t; i < M.n_par; i += nt) pb[i] = M.p_tpl[i];
  __syncthreads();                    // (the template row is in place)
  if (t != 0) return;
  for (int c = 0; c < nd; ++c) {
    pb[M.p_state0 + c] = s0[c];
    pb[M.p_input0 + c] = u0[c];
    pb[M.p_poseT + c] = stT[c];
  }
  omg_mpc_write_obstacles(M, b, obs, pb);
}

// The rows that are not stopped, in ascending order, and their count: one block, a scan per chunk
// of blockDim rows.  Shared memory: [blockDim] ints.
__global__ void omg_mpc_rows_kernel(int B, const int* __restrict__ stop, int* __restrict__ rows, int* __restrict__ n_rows) {
  OMG_DYN_SHARED(scd);
  int* sc = reinterpret_cast<int*>(scd);
  const int t = threadIdx.x, nt = blockDim.x;
  int base = 0;
  for (int c0 = 0; c0 < B; c0 += nt) {
    const int live = (c0 + t < B && !stop[c0 + t]) ? 1 : 0;
    sc[t] = live;
    __syncthreads();
    for (int d = 1; d < nt; d *= 2) {         // inclusive scan (Hillis-Steele)
      const int v = t >= d ? sc[t - d] : 0;
      __syncthreads();
      sc[t] += v;
      __syncthreads();
    }
    if (live) rows[base + sc[t] - 1] = c0 + t;
    base += sc[nt - 1];
    __syncthreads();
  }
  if (t == 0) *n_rows = base;
}

// Free motion time, shared memory as omg_mpc_commit_kernel.  A stopped instance reads nothing of the
// solve: status -1, 0 iterations.  Status 0: the row takes the solution, the output rows are the
// plan at min(j sample_time, T) / T, and the next prediction's samples are stored (ideal: at
// min(update_time, T) / T; integrate: s sample_time / T for s <= round6(min(update_time, T) /
// sample_time)).  Any other status keeps the warm start it was solved from.
__global__ void omg_mpc_commit_free_kernel(const MpcDev M, int* __restrict__ status, int* __restrict__ iters,
                                           double* __restrict__ state_traj, double* __restrict__ input_traj) {
  OMG_DYN_SHARED(cd);
  const int b = blockIdx.x, t = threadIdx.x, nt = blockDim.x, n = M.n, nd = M.nd, L = M.L, p = M.p;
  if (b >= M.B) return;
  if (M.stop[b]) {
    if (t == 0) { status[b] = -1; iters[b] = 0; }
    return;
  }
  const bool ok = status[b] == 0;
  const double* src = (ok ? M.Xn : M.X0) + (size_t)b * n;
  double* xb = M.X + (size_t)b * n;
  for (int i = t; i < n; i += nt) xb[i] = src[i];
  if (!ok) {                          // keep the warm start; a cold start stays one
    if (t == 0 && M.phase[b] != OMG_MPC_COLD) M.phase[b] = OMG_MPC_FAILED;
    return;
  }
  for (int c = t; c < nd; c += nt) omg_spl_der_coef(M.knots, p, L, 2, src + M.spl_off + c * L, cd + (size_t)c * 2 * L);
  __syncthreads();
  const double T = src[M.t_index], st = M.sample_time;
  const bool ideal = M.mode == OMG_MPC_PREDICT_IDEAL;
  const int ns = (int)omg_round6(fmin(M.update_time, T) / st);
  const int tl = M.traj_len, n_pts = tl + (ideal ? 1 : ns + 1);
  for (int j = t; j < n_pts; j += nt) {
    const double tau = j < tl ? fmin((double)j * st, T) / T
                       : ideal ? fmin(M.update_time, T) / T : (double)(j - tl) * st / T;
    double w[OMG_SPL_MAX_LEN + OMG_SPL_MAX_DEGREE], v[2][OMG_CL_MAX_INPUT];
    for (int d = 0; d < 2; ++d) {
      omg_cox_de_boor(M.knots + d, p - d, tau, 0, L - d, w);
      for (int c = 0; c < nd; ++c) {
        const double* q = cd + ((size_t)c * 2 + d) * L;
        double acc = 0.0;
        for (int i = 0; i < L - d; ++i) acc += w[i] * q[i];
        v[d][c] = d ? acc / T : acc;
      }
    }
    double *xo, *uo;
    if (j < tl) {
      xo = state_traj + ((size_t)b * tl + j) * nd;
      uo = input_traj + ((size_t)b * tl + j) * nd;
    } else if (ideal) {
      xo = M.pred_x + (size_t)b * nd;
      uo = M.pred_u + (size_t)b * nd;
    } else {
      xo = nullptr;
      uo = M.U + ((size_t)b * (M.n_samp + 1) + (j - tl)) * nd;
    }
    for (int c = 0; c < nd; ++c) {
      if (xo) xo[c] = v[0][c];
      uo[c] = v[1][c];
    }
  }
  __syncthreads();                    // (every thread has read t_b)
  if (t == 0) {
    M.Tm[b] = T;
    M.ns[b] = ns;
    M.phase[b] = OMG_MPC_ACCEPTED;
    M.t[b] = omg_round6(M.t[b] + M.update_time);
  }
}

__global__ void omg_mpc_fill_kernel(int B, double v, double* __restrict__ out) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < B) out[b] = v;
}

__global__ void omg_mpc_flag_kernel(int B, const int* __restrict__ mask, int* __restrict__ rec) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < B && mask[b]) rec[b] = 1;
}

// One instance per block: store its shape record and rewrite the rows of its obstacles in its bound
// row, the tables' bounds lbg / ubg where avoid is set and -inf / +inf where it is not (updateBounds).
__global__ void omg_mpc_set_obstacles_kernel(const MpcDev M, const double* __restrict__ shapes,
                                             const int* __restrict__ avoid, const double* __restrict__ lbg,
                                             const double* __restrict__ ubg) {
  const int b = blockIdx.x, t = threadIdx.x, nt = blockDim.x;
  if (b >= M.B) return;
  if (shapes)
    for (int i = t; i < M.n_shape; i += nt) M.shapes[(size_t)b * M.n_shape + i] = shapes[(size_t)b * M.n_shape + i];
  if (!avoid) return;
  double* lb = M.lbg + (size_t)b * M.m;
  double* ub = M.ubg + (size_t)b * M.m;
  for (int k = 0; k < M.n_obs; ++k) {
    const int* g = M.obs_geo + 6 * k;
    const bool on = avoid[(size_t)b * M.n_obs + k] != 0;
    for (int r = g[4] + t; r < g[4] + g[5]; r += nt) {
      lb[r] = on ? lbg[r] : -INFINITY;
      ub[r] = on ? ubg[r] : INFINITY;
    }
  }
}

#define OMG_MPC_NT 128

struct omg_mpc {
  omg_problem* h = nullptr;
  bool free_T = false;
  MpcDev M;
  size_t smem_prepare = 0, smem_commit = 0;
  std::vector<void*> allocs;
  double* lam = nullptr; double* f = nullptr;
  int* mask = nullptr;
  // device staging of omg_mpc_update_host
  double *s0 = nullptr, *sT = nullptr, *obs = nullptr, *xtraj = nullptr, *utraj = nullptr;
  int *st = nullptr, *it = nullptr;
  // device staging of omg_mpc_set_obstacles_host (allocated by omg_mpc_attach_obstacles)
  double* hshapes = nullptr; int* havoid = nullptr;
};

namespace {
// fields of an MPC file: kind 0 int32 scalar, 1 float64 scalar, 2 int32 array, 3 float64 array
struct MpcField { const char* name; int kind; size_t off; };
#define MF(f, k) {#f, k, offsetof(omg_mpc_desc, f)}
const MpcField kMpcFields[] = {
  MF(n, 0), MF(n_par, 0), MF(n_dim, 0), MF(spl_offset, 0), MF(L, 0), MF(degree, 0), MF(knots, 3),
  MF(horizon, 1), MF(knot_time, 1), MF(update_time, 1), MF(sample_time, 1),
  MF(p_state0, 0), MF(p_input0, 0), MF(p_poseT, 0), MF(p_t, 0), MF(p_T, 0),
  MF(n_obs, 0), MF(obs_kind, 2), MF(obs_off, 2),
  MF(n_shift, 0), MF(shift_off, 2), MF(shift_len, 2), MF(shift_ncol, 2), MF(shift_T, 3),
  MF(x_template, 3), MF(p_template, 3),
};
#undef MF
#define MF(f, k) {#f, k, offsetof(omg_mpc_freeT_desc, f)}
const MpcField kMpcFreeTFields[] = {
  MF(n, 0), MF(n_par, 0), MF(n_dim, 0), MF(spl_offset, 0), MF(L, 0), MF(degree, 0), MF(knots, 3),
  MF(update_time, 1), MF(sample_time, 1), MF(stop_tol, 1), MF(t_index, 0),
  MF(p_state0, 0), MF(p_input0, 0), MF(p_poseT, 0),
  MF(n_obs, 0), MF(obs_kind, 2), MF(obs_off, 2),
  MF(n_blocks, 0), MF(blk_off, 2), MF(blk_len, 2), MF(blk_ncol, 2), MF(blk_degree, 2), MF(blk_knots, 3),
  MF(x_template, 3), MF(p_template, 3),
};
#undef MF
#define MF(f, k) {#f, k, offsetof(omg_mpc_obstacles_desc, f)}
const MpcField kMpcObstacleFields[] = {
  MF(n_obs, 0), MF(chk_off, 2), MF(chk_len, 2), MF(rad_off, 2), MF(rad_len, 2), MF(row_off, 2), MF(row_len, 2),
};
#undef MF
template <class D> struct OwnedDesc { D desc; std::vector<void*> blocks; };

// A file of the record container with magic `magic` (`what`: its name in messages) of the fields
// `fields` into a heap descriptor; a record that is not one of them but one of `other` (no) marks the
// other kind of MPC file, which `other_reader` reads.
template <class D>
D* mpc_read_file(const char* path, const MpcField* fields, int nf, const MpcField* other, int no,
                 const char* other_reader, const char* magic_ = "OMGMPC\0\0", const std::string& what = "MPC") {
  FILE* fp = path ? fopen(path, "rb") : nullptr;
  if (!fp) { set_err("cannot open " + what + " file " + (path ? path : "(null)")); return nullptr; }
  OwnedDesc<D>* O = new OwnedDesc<D>();
  memset(&O->desc, 0, sizeof(O->desc));
  bool ok = true;
  char magic[8]; int32_t ver = 0, nrec = 0;
  if (fread(magic, 1, 8, fp) != 8 || memcmp(magic, magic_, 8) != 0) { set_err("not an omg " + what + " file"); ok = false; }
  if (ok && (fread(&ver, 4, 1, fp) != 1 || fread(&nrec, 4, 1, fp) != 1)) { set_err("truncated " + what + " file"); ok = false; }
  if (ok && ver != OMG_ABI_VERSION) { set_err(what + " file written for another ABI version"); ok = false; }
  std::vector<char> seen(nf, 0);
  for (int r = 0; ok && r < nrec; ++r) {
    char name[24]; int32_t dtype = 0, pad = 0; int64_t count = 0;
    if (fread(name, 1, 24, fp) != 24 || fread(&dtype, 4, 1, fp) != 1 || fread(&pad, 4, 1, fp) != 1 ||
        fread(&count, 8, 1, fp) != 1 || count < 0) { set_err("truncated " + what + " file"); ok = false; break; }
    name[23] = 0;
    int k = -1;
    for (int q = 0; q < nf; ++q) if (strcmp(fields[q].name, name) == 0) { k = q; break; }
    bool other_kind = false;
    for (int q = 0; k < 0 && q < no; ++q) other_kind = other_kind || strcmp(other[q].name, name) == 0;
    if (other_kind) {
      set_err(std::string("this MPC file is of the other kind: read it with ") + other_reader); ok = false; break; }
    const int kind = k < 0 ? -1 : fields[k].kind;
    if (k < 0 || dtype != (kind == 1 || kind == 3 ? 1 : 0)) { set_err("unknown record in " + what + " file: " + name); ok = false; break; }
    const size_t esz = dtype ? 8 : 4;
    char* base = reinterpret_cast<char*>(&O->desc) + fields[k].off;
    if (kind < 2) {
      if (count != 1 || fread(base, esz, 1, fp) != 1) { set_err(std::string("bad scalar record ") + name); ok = false; break; }
    } else {
      void* blk = malloc((size_t)(count > 0 ? count : 1) * esz);
      O->blocks.push_back(blk);
      if (!blk || (count > 0 && fread(blk, esz, (size_t)count, fp) != (size_t)count)) { set_err("truncated " + what + " file"); ok = false; break; }
      *reinterpret_cast<void**>(base) = blk;
    }
    seen[k] = 1;
  }
  fclose(fp);
  for (int q = 0; ok && q < nf; ++q)
    if (!seen[q]) { set_err(what + " file lacks " + fields[q].name); ok = false; }
  if (!ok) { for (void* b : O->blocks) free(b); delete O; return nullptr; }
  return &O->desc;
}

template <class D> void mpc_free_file(D* desc) {
  if (!desc) return;
  OwnedDesc<D>* O = reinterpret_cast<OwnedDesc<D>*>(desc);   // desc is the first member
  for (void* b : O->blocks) free(b);
  delete O;
}

bool mpc_range(const std::string& f, const std::string& what, int64_t lo, int64_t len, int64_t size) {
  if (lo < 0 || len < 0 || lo + len > size) {
    set_err(f + what + " at " + std::to_string(lo) + " (+" + std::to_string(len) + ") outside [0, " +
            std::to_string(size) + ")");
    return false;
  }
  return true;
}

// The checks both kinds of descriptor share (f: the message prefix); n_samp receives
// update_time / sample_time.
template <class D>
bool mpc_check_common(const std::string& f, const omg_problem* h, const D* d, int32_t B, int32_t mode, int* n_samp) {
  if (d->n != h->T.n || d->n_par != h->T.n_par) {
    set_err(f + "the descriptor is for n = " + std::to_string(d->n) + ", n_par = " + std::to_string(d->n_par) +
            ", the problem has n = " + std::to_string(h->T.n) + ", n_par = " + std::to_string(h->T.n_par));
    return false;
  }
  if (B <= 0) { set_err(f + "B must be >= 1, got " + std::to_string(B)); return false; }
  if (mode != OMG_MPC_PREDICT_IDEAL && mode != OMG_MPC_PREDICT_INTEGRATE) {
    set_err(f + "unknown prediction " + std::to_string(mode)); return false; }
  if (!(d->sample_time > 0.0) || !(d->update_time > 0.0)) {
    set_err(f + "update_time and sample_time must be > 0"); return false; }
  const double r = d->update_time / d->sample_time;
  *n_samp = (int)rint(r);
  if (*n_samp < 1 || fabs(r - *n_samp) > 1e-9 * std::max(1.0, r)) {
    set_err(f + "update_time " + std::to_string(d->update_time) + " is not a multiple of sample_time " +
            std::to_string(d->sample_time)); return false; }
  const int nd = d->n_dim, L = d->L, p = d->degree;
  if (nd < 1 || nd > OMG_CL_MAX_INPUT) { set_err(f + "n_dim must be 1 .. 3"); return false; }
  if (p < 1 || p > OMG_SPL_MAX_DEGREE || L < p + 1 || L > OMG_SPL_MAX_LEN) {
    set_err(f + "degree " + std::to_string(p) + " / basis length " + std::to_string(L) + " outside 1 <= p <= " +
            std::to_string(OMG_SPL_MAX_DEGREE) + ", p + 1 <= L <= " + std::to_string(OMG_SPL_MAX_LEN)); return false; }
  if (!d->knots || !d->x_template || !d->p_template || (d->n_obs > 0 && (!d->obs_kind || !d->obs_off)) ||
      d->n_obs < 0) { set_err(f + "null descriptor array"); return false; }
  for (int j = 0; j < L + p; ++j)
    if (!(d->knots[j] <= d->knots[j + 1])) { set_err(f + "knots not non-decreasing"); return false; }
  if (!mpc_range(f, "vehicle splines", d->spl_offset, (int64_t)nd * L, d->n) ||
      !mpc_range(f, "state0", d->p_state0, nd, d->n_par) || !mpc_range(f, "input0", d->p_input0, nd, d->n_par) ||
      !mpc_range(f, "poseT", d->p_poseT, nd, d->n_par)) return false;
  for (int k = 0; k < d->n_obs; ++k) {
    const std::string o = "obstacle " + std::to_string(k) + " ";
    if (d->obs_kind[k] != 0 && d->obs_kind[k] != 1) { set_err(f + o + "kind must be 0 or 1"); return false; }
    for (int q = 0; q < 3; ++q)
      if (!mpc_range(f, o + "x/v/a", d->obs_off[4 * k + q], nd, d->n_par)) return false;
    if (d->obs_kind[k] && !mpc_range(f, o + "theta", d->obs_off[4 * k + 3], 1, d->n_par)) return false;
  }
  return true;
}

// Checks of omg_mpc_create; n_samp receives update_time / sample_time.
bool mpc_check(const omg_problem* h, const omg_mpc_desc* D, int32_t B, int32_t traj_len, int32_t mode, int* n_samp) {
  const std::string f("omg_mpc_create: ");
  if (!(D->horizon > 0.0) || !(D->knot_time > 0.0) || !(D->sample_time > 0.0) || !(D->update_time > 0.0)) {
    set_err(f + "horizon, knot_time, update_time and sample_time must be > 0"); return false; }
  if (!mpc_check_common(f, h, D, B, mode, n_samp)) return false;
  const int max_len = (int)rint(D->horizon / D->sample_time * 1e6) / 1000000;
  if (traj_len < 1 || traj_len > max_len) {
    set_err(f + "trajectory_length " + std::to_string(traj_len) + " outside 1 .. horizon / sample_time = " +
            std::to_string(max_len)); return false; }
  if ((D->n_shift > 0 && (!D->shift_off || !D->shift_len || !D->shift_ncol || !D->shift_T)) || D->n_shift < 0) {
    set_err(f + "null descriptor array"); return false; }
  if (!mpc_range(f, "t", D->p_t, 1, D->n_par) || !mpc_range(f, "T", D->p_T, 1, D->n_par)) return false;
  for (int k = 0; k < D->n_shift; ++k)
    if (D->shift_len[k] < 1 || D->shift_ncol[k] < 1 ||
        !mpc_range(f, "shift block " + std::to_string(k), D->shift_off[k], (int64_t)D->shift_len[k] * D->shift_ncol[k], D->n))
      return false;
  if (2 * (size_t)D->n * sizeof(double) > 227 * 1024) { set_err(f + "two x rows exceed the shared memory of a block"); return false; }
  return true;
}

// Checks of omg_mpc_create_freet; n_samp as above, iv / n_knots / Lmax / pmax: the block
// descriptor of spline_desc.
bool mpc_check_freeT(const omg_problem* h, const omg_mpc_freeT_desc* D, int32_t B, int32_t traj_len, int32_t mode,
                     int* n_samp, std::vector<int>& iv, size_t* n_knots, int* Lmax, int* pmax) {
  const std::string f("omg_mpc_create_freet: ");
  if (!mpc_check_common(f, h, D, B, mode, n_samp)) return false;
  if (!(D->stop_tol >= 0.0)) { set_err(f + "stop_tol must be >= 0"); return false; }
  if (D->t_index < 0 || D->t_index >= D->n) {
    set_err(f + "t_index " + std::to_string(D->t_index) + " outside [0, " + std::to_string(D->n) + ")"); return false; }
  const double T = D->x_template[D->t_index];
  const int max_len = T > 0.0 ? (int)rint(T / D->sample_time * 1e6) / 1000000 : 0;
  if (traj_len < 1 || traj_len > max_len) {
    set_err(f + "trajectory_length " + std::to_string(traj_len) + " outside 1 .. (template T) / sample_time = " +
            std::to_string(max_len)); return false; }
  if (D->n_blocks < 0 || (D->n_blocks > 0 && (!D->blk_off || !D->blk_len || !D->blk_ncol || !D->blk_degree ||
                                              !D->blk_knots))) { set_err(f + "null descriptor array"); return false; }
  size_t n_coef = 0;
  if (!spline_desc("omg_mpc_create_freet", D->n, D->n_blocks, D->blk_off, D->blk_len, D->blk_ncol, D->blk_degree,
                   D->blk_knots, 1, iv, n_knots, Lmax, pmax, &n_coef)) return false;
  const size_t smem = sizeof(double) * (2 * (size_t)D->n + 2 * (size_t)*Lmax + *pmax + 1 + 2 * OMG_MPC_NT +
                                        2 * (size_t)*Lmax * *Lmax);
  if (smem > 227 * 1024) { set_err(f + "two x rows and the shift's bases exceed the shared memory of a block"); return false; }
  return true;
}
}  // namespace

extern "C" {

omg_mpc_desc* omg_mpc_read(const char* path) {
  const int nf = (int)(sizeof(kMpcFields) / sizeof(kMpcFields[0]));
  const int no = (int)(sizeof(kMpcFreeTFields) / sizeof(kMpcFreeTFields[0]));
  return mpc_read_file<omg_mpc_desc>(path, kMpcFields, nf, kMpcFreeTFields, no, "omg_mpc_freet_read");
}

void omg_mpc_free_desc(omg_mpc_desc* desc) { mpc_free_file(desc); }

omg_mpc_freeT_desc* omg_mpc_freet_read(const char* path) {
  const int nf = (int)(sizeof(kMpcFreeTFields) / sizeof(kMpcFreeTFields[0]));
  const int no = (int)(sizeof(kMpcFields) / sizeof(kMpcFields[0]));
  return mpc_read_file<omg_mpc_freeT_desc>(path, kMpcFreeTFields, nf, kMpcFields, no, "omg_mpc_read");
}

void omg_mpc_freet_release(omg_mpc_freeT_desc* desc) { mpc_free_file(desc); }

void omg_mpc_destroy(omg_mpc* mpc) {
  if (!mpc) return;
  cudaSetDevice(mpc->h->device);
  for (void* p : mpc->allocs) cudaFree(p);
  delete mpc;
}

}  // extern "C"

namespace {
// A device buffer of the handle, a copy of src (or zeros); *ok turns false on failure.
void* mpc_alloc(omg_mpc* q, size_t bytes, const void* src, bool* ok) {
  void* d = nullptr;
  if (cudaMalloc(&d, bytes ? bytes : 8) != cudaSuccess) { *ok = false; return nullptr; }
  q->allocs.push_back(d);
  if (src && bytes && cudaMemcpy(d, src, bytes, cudaMemcpyHostToDevice) != cudaSuccess) *ok = false;
  else if (!src && cudaMemset(d, 0, bytes ? bytes : 8) != cudaSuccess) *ok = false;
  return d;
}

// The handle's fields and buffers both kinds of descriptor share.
template <class D>
omg_mpc* mpc_new(omg_problem* h, const D* d, int32_t B, int32_t traj_len, int32_t mode, int n_samp, bool* ok) {
  omg_mpc* q = new omg_mpc();
  q->h = h;
  MpcDev& M = q->M;
  memset(&M, 0, sizeof(M));
  const int n = d->n, np_ = d->n_par, nd = d->n_dim, L = d->L, p = d->degree;
  M.B = B; M.n = n; M.n_par = np_; M.nd = nd; M.spl_off = d->spl_offset; M.L = L; M.p = p;
  M.traj_len = traj_len; M.n_samp = n_samp; M.mode = mode; M.n_obs = d->n_obs;
  M.p_state0 = d->p_state0; M.p_input0 = d->p_input0; M.p_poseT = d->p_poseT;
  M.update_time = d->update_time; M.sample_time = d->sample_time;
  const size_t b = B, d8 = sizeof(double);
  M.knots = (const double*)mpc_alloc(q, d8 * (L + p + 1), d->knots, ok);
  M.obs_kind = (const int*)mpc_alloc(q, 4 * (size_t)d->n_obs, d->obs_kind, ok);
  M.obs_off = (const int*)mpc_alloc(q, 16 * (size_t)d->n_obs, d->obs_off, ok);
  M.x_tpl = (const double*)mpc_alloc(q, d8 * n, d->x_template, ok);
  M.p_tpl = (const double*)mpc_alloc(q, d8 * np_, d->p_template, ok);
  M.X = (double*)mpc_alloc(q, d8 * b * n, nullptr, ok);
  M.X0 = (double*)mpc_alloc(q, d8 * b * n, nullptr, ok);
  M.Xn = (double*)mpc_alloc(q, d8 * b * n, nullptr, ok);
  M.P = (double*)mpc_alloc(q, d8 * b * np_, nullptr, ok);
  M.t = (double*)mpc_alloc(q, d8 * b, nullptr, ok);
  M.pred_x = (double*)mpc_alloc(q, d8 * b * nd, nullptr, ok);
  M.pred_u = (double*)mpc_alloc(q, d8 * b * nd, nullptr, ok);
  M.U = (double*)mpc_alloc(q, d8 * b * (n_samp + 1) * nd, nullptr, ok);
  M.rec = (int*)mpc_alloc(q, 4 * b, nullptr, ok);
  q->lam = (double*)mpc_alloc(q, d8 * b * h->T.m, nullptr, ok);
  q->f = (double*)mpc_alloc(q, d8 * b, nullptr, ok);
  q->mask = (int*)mpc_alloc(q, 4 * b, nullptr, ok);
  q->s0 = (double*)mpc_alloc(q, d8 * b * nd, nullptr, ok);
  q->sT = (double*)mpc_alloc(q, d8 * b * nd, nullptr, ok);
  q->obs = (double*)mpc_alloc(q, d8 * b * d->n_obs * (3 * nd + 1), nullptr, ok);
  q->xtraj = (double*)mpc_alloc(q, d8 * b * traj_len * nd, nullptr, ok);
  q->utraj = (double*)mpc_alloc(q, d8 * b * traj_len * nd, nullptr, ok);
  q->st = (int*)mpc_alloc(q, 4 * b, nullptr, ok);
  q->it = (int*)mpc_alloc(q, 4 * b, nullptr, ok);
  q->smem_commit = 2 * d8 * nd * L;
  return q;
}
}  // namespace

extern "C" {

omg_mpc* omg_mpc_create(omg_problem* h, const omg_mpc_desc* D, int32_t B, int32_t traj_len, int32_t mode) {
  if (!h || !D) { set_err("omg_mpc_create: null argument"); return nullptr; }
  int n_samp = 0;
  if (!mpc_check(h, D, B, traj_len, mode, &n_samp)) return nullptr;
  if (cudaSetDevice(h->device) != cudaSuccess) { set_err("omg_mpc_create: cudaSetDevice failed"); return nullptr; }
  bool ok = true;
  omg_mpc* q = mpc_new(h, D, B, traj_len, mode, n_samp, &ok);
  MpcDev& M = q->M;
  M.n_shift = D->n_shift; M.p_t = D->p_t; M.p_T = D->p_T;
  M.horizon = D->horizon; M.knot_time = D->knot_time;
  std::vector<int> sd(4 * (size_t)D->n_shift);
  size_t nT = 0;
  for (int k = 0; k < D->n_shift; ++k) {
    sd[4 * k] = D->shift_off[k]; sd[4 * k + 1] = D->shift_len[k]; sd[4 * k + 2] = D->shift_ncol[k]; sd[4 * k + 3] = (int)nT;
    nT += (size_t)D->shift_len[k] * D->shift_len[k];
  }
  M.shift_desc = (const int*)mpc_alloc(q, 4 * sd.size(), sd.data(), &ok);
  M.shift_T = (const double*)mpc_alloc(q, sizeof(double) * nT, D->shift_T, &ok);
  M.t_prev = (double*)mpc_alloc(q, sizeof(double) * B, nullptr, &ok);
  q->smem_prepare = 2 * sizeof(double) * D->n;
  if (ok && q->smem_prepare > 48 * 1024 &&
      cudaFuncSetAttribute((const void*)omg_mpc_prepare_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                           (int)q->smem_prepare) != cudaSuccess) ok = false;
  if (!ok) { set_err("omg_mpc_create: device allocation/upload failed"); omg_mpc_destroy(q); return nullptr; }
  return q;
}

omg_mpc* omg_mpc_create_freet(omg_problem* h, const omg_mpc_freeT_desc* D, int32_t B, int32_t traj_len, int32_t mode) {
  if (!h || !D) { set_err("omg_mpc_create_freet: null argument"); return nullptr; }
  int n_samp = 0, Lmax = 1, pmax = 0;
  std::vector<int> iv;
  size_t n_knots = 0;
  if (!mpc_check_freeT(h, D, B, traj_len, mode, &n_samp, iv, &n_knots, &Lmax, &pmax)) return nullptr;
  if (cudaSetDevice(h->device) != cudaSuccess) { set_err("omg_mpc_create_freet: cudaSetDevice failed"); return nullptr; }
  bool ok = true;
  omg_mpc* q = mpc_new(h, D, B, traj_len, mode, n_samp, &ok);
  q->free_T = true;
  MpcDev& M = q->M;
  M.t_index = D->t_index; M.n_blocks = D->n_blocks; M.Lmax = Lmax; M.pmax = pmax; M.stop_tol = D->stop_tol;
  M.blk_desc = (const int*)mpc_alloc(q, 4 * iv.size(), iv.data(), &ok);
  M.blk_knots = (const double*)mpc_alloc(q, sizeof(double) * n_knots, D->blk_knots, &ok);
  const std::vector<double> T0(B, D->x_template[D->t_index]);
  M.Tm = (double*)mpc_alloc(q, sizeof(double) * B, T0.data(), &ok);
  M.phase = (int*)mpc_alloc(q, 4 * (size_t)B, nullptr, &ok);
  M.stop = (int*)mpc_alloc(q, 4 * (size_t)B, nullptr, &ok);
  M.ns = (int*)mpc_alloc(q, 4 * (size_t)B, nullptr, &ok);
  M.rows = (int*)mpc_alloc(q, 4 * (size_t)B, nullptr, &ok);
  M.n_rows = (int*)mpc_alloc(q, 4, nullptr, &ok);
  q->smem_prepare = sizeof(double) * (2 * (size_t)D->n + 2 * (size_t)Lmax + pmax + 1 + 2 * OMG_MPC_NT +
                                      2 * (size_t)Lmax * Lmax);
  if (ok && q->smem_prepare > 48 * 1024 &&
      cudaFuncSetAttribute((const void*)omg_mpc_prepare_free_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                           (int)q->smem_prepare) != cudaSuccess) ok = false;
  if (!ok) { set_err("omg_mpc_create_freet: device allocation/upload failed"); omg_mpc_destroy(q); return nullptr; }
  return q;
}

int omg_mpc_update(omg_mpc* q, const double* state0, const double* stateT, const double* obstacles,
                   double* state_traj, double* input_traj, int32_t* status, int32_t* iters, void* stream_) {
  if (!q || !state0 || !stateT || (q && q->M.n_obs > 0 && !obstacles) || !state_traj || !input_traj || !status ||
      !iters) { set_err("omg_mpc_update: null argument"); return -1; }
  cudaStream_t stream = (cudaStream_t)stream_;
  omg_problem* h = q->h;
  CK(cudaSetDevice(h->device));
  const int B = q->M.B;
  // the tables' bounds, shared by every instance, or with obstacles attached each instance's own row
  const bool own = q->M.shapes != nullptr;
  const double* lbg = own ? q->M.lbg : h->lbg;
  const double* ubg = own ? q->M.ubg : h->ubg;
  const int32_t shared = own ? 0 : 1;
  if (q->free_T) {
    OMG_LAUNCH(omg_mpc_prepare_free_kernel, B, OMG_MPC_NT, q->smem_prepare, stream, q->M, state0, stateT, obstacles);
    CK(cudaGetLastError());
    OMG_LAUNCH(omg_mpc_rows_kernel, 1, 256, 256 * sizeof(int), stream, B, q->M.stop, q->M.rows, q->M.n_rows);
    CK(cudaGetLastError());
    if (solve_batch_rows(h, B, q->M.X0, q->M.P, lbg, ubg, shared, nullptr, q->M.Xn, q->lam, q->f, status, iters,
                         q->M.rows, q->M.n_rows, stream))
      return -1;
    OMG_LAUNCH(omg_mpc_commit_free_kernel, B, OMG_MPC_NT, q->smem_commit, stream, q->M, status, iters, state_traj,
               input_traj);
    CK(cudaGetLastError());
    return 0;
  }
  OMG_LAUNCH(omg_mpc_prepare_kernel, B, OMG_MPC_NT, q->smem_prepare, stream, q->M, state0, stateT, obstacles);
  CK(cudaGetLastError());
  if (omg_solve_batch(h, B, q->M.X0, q->M.P, lbg, ubg, shared, nullptr, q->M.Xn, q->lam, q->f, status, iters, stream))
    return -1;
  OMG_LAUNCH(omg_mpc_commit_kernel, B, OMG_MPC_NT, q->smem_commit, stream, q->M, status, state_traj, input_traj);
  CK(cudaGetLastError());
  return 0;
}

int omg_mpc_update_host(omg_mpc* q, const double* state0, const double* stateT, const double* obstacles,
                        double* state_traj, double* input_traj, int32_t* status, int32_t* iters) {
  if (!q || !state0 || !stateT || (q && q->M.n_obs > 0 && !obstacles) || !state_traj || !input_traj || !status ||
      !iters) { set_err("omg_mpc_update_host: null argument"); return -1; }
  CK(cudaSetDevice(q->h->device));
  const size_t b = q->M.B, nd = q->M.nd, no = (size_t)q->M.n_obs * (3 * nd + 1), nt = (size_t)q->M.traj_len * nd;
  CK(cudaMemcpy(q->s0, state0, b * nd * 8, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(q->sT, stateT, b * nd * 8, cudaMemcpyHostToDevice));
  if (no) CK(cudaMemcpy(q->obs, obstacles, b * no * 8, cudaMemcpyHostToDevice));
  // (the rows of a failed solve keep what the caller's buffers hold)
  CK(cudaMemcpy(q->xtraj, state_traj, b * nt * 8, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(q->utraj, input_traj, b * nt * 8, cudaMemcpyHostToDevice));
  if (omg_mpc_update(q, q->s0, q->sT, q->obs, q->xtraj, q->utraj, q->st, q->it, nullptr)) return -1;
  CK(cudaMemcpy(state_traj, q->xtraj, b * nt * 8, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(input_traj, q->utraj, b * nt * 8, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(status, q->st, b * 4, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(iters, q->it, b * 4, cudaMemcpyDeviceToHost));
  return 0;
}

int omg_mpc_recover(omg_mpc* q, const int32_t* mask) {
  if (!q || !mask) { set_err("omg_mpc_recover: null argument"); return -1; }
  CK(cudaSetDevice(q->h->device));
  CK(cudaMemcpy(q->mask, mask, (size_t)q->M.B * 4, cudaMemcpyHostToDevice));
  OMG_LAUNCH(omg_mpc_flag_kernel, (q->M.B + 127) / 128, 128, 0, nullptr, q->M.B, q->mask, q->M.rec);
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(nullptr));
  return 0;
}

int omg_mpc_time(omg_mpc* q, double* t_out) {
  if (!q || !t_out) { set_err("omg_mpc_time: null argument"); return -1; }
  CK(cudaSetDevice(q->h->device));
  CK(cudaDeviceSynchronize());
  CK(cudaMemcpy(t_out, q->M.t, (size_t)q->M.B * 8, cudaMemcpyDeviceToHost));
  return 0;
}

int omg_mpc_motion_time(omg_mpc* q, double* T_out, void* stream_) {
  if (!q || !T_out) { set_err("omg_mpc_motion_time: null argument"); return -1; }
  cudaStream_t stream = (cudaStream_t)stream_;
  CK(cudaSetDevice(q->h->device));
  const int B = q->M.B;
  if (q->free_T) CK(cudaMemcpyAsync(T_out, q->M.Tm, (size_t)B * 8, cudaMemcpyDeviceToDevice, stream));
  else {
    OMG_LAUNCH(omg_mpc_fill_kernel, (B + 127) / 128, 128, 0, stream, B, q->M.horizon, T_out);
    CK(cudaGetLastError());
  }
  return 0;
}

int omg_mpc_last_problem(omg_mpc* q, double* x0_out, double* p_out, void* stream_) {
  if (!q) { set_err("omg_mpc_last_problem: null argument"); return -1; }
  cudaStream_t stream = (cudaStream_t)stream_;
  CK(cudaSetDevice(q->h->device));
  const size_t b = q->M.B;
  if (x0_out) CK(cudaMemcpyAsync(x0_out, q->M.X0, b * q->M.n * 8, cudaMemcpyDeviceToDevice, stream));
  if (p_out) CK(cudaMemcpyAsync(p_out, q->M.P, b * q->M.n_par * 8, cudaMemcpyDeviceToDevice, stream));
  return 0;
}

omg_mpc_obstacles_desc* omg_mpc_obstacles_read(const char* path) {
  const int nf = (int)(sizeof(kMpcObstacleFields) / sizeof(kMpcObstacleFields[0]));
  return mpc_read_file<omg_mpc_obstacles_desc>(path, kMpcObstacleFields, nf, nullptr, 0, "", "OMGOBS\0\0", "obstacle");
}

void omg_mpc_obstacles_release(omg_mpc_obstacles_desc* desc) { mpc_free_file(desc); }

int omg_mpc_attach_obstacles(omg_mpc* q, const omg_mpc_obstacles_desc* D) {
  const std::string f("omg_mpc_attach_obstacles: ");
  if (!q || !D) { set_err(f + "null argument"); return -1; }
  MpcDev& M = q->M;
  if (M.shapes) { set_err(f + "this handle already has obstacles attached"); return -1; }
  if (D->n_obs != M.n_obs) {
    set_err(f + "the descriptor has " + std::to_string(D->n_obs) + " obstacles, the handle " + std::to_string(M.n_obs));
    return -1;
  }
  const int n_obs = M.n_obs, m = q->h->T.m, np_ = M.n_par;
  if (n_obs > 0 && (!D->chk_off || !D->chk_len || !D->rad_off || !D->rad_len || !D->row_off || !D->row_len)) {
    set_err(f + "null descriptor array"); return -1; }
  CK(cudaSetDevice(q->h->device));
  std::vector<double> lbg(m), ubg(m), ptpl(np_);
  CK(cudaMemcpy(lbg.data(), q->h->lbg, (size_t)m * 8, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(ubg.data(), q->h->ubg, (size_t)m * 8, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(ptpl.data(), M.p_tpl, (size_t)np_ * 8, cudaMemcpyDeviceToHost));
  std::vector<int> geo(6 * (size_t)n_obs);
  std::vector<char> taken(m, 0);
  std::vector<double> rec;                 // one instance's shape record: the template's shapes
  for (int k = 0; k < n_obs; ++k) {
    const std::string o = "obstacle " + std::to_string(k) + " ";
    if (!mpc_range(f, o + "checkpoints", D->chk_off[k], D->chk_len[k], np_) ||
        !mpc_range(f, o + "radii", D->rad_off[k], D->rad_len[k], np_) ||
        !mpc_range(f, o + "rows", D->row_off[k], D->row_len[k], m)) return -1;
    if (D->rad_len[k] < 1 || D->chk_len[k] != M.nd * D->rad_len[k]) {
      set_err(f + o + "has " + std::to_string(D->chk_len[k]) + " checkpoint coordinates and " +
              std::to_string(D->rad_len[k]) + " radii; n_dim = " + std::to_string(M.nd) + " coordinates per radius");
      return -1;
    }
    for (int r = D->row_off[k]; r < D->row_off[k] + D->row_len[k]; ++r) {
      if (taken[r]) { set_err(f + o + "rows overlap another obstacle's at row " + std::to_string(r)); return -1; }
      if (lbg[r] == ubg[r]) {
        set_err(f + o + "row " + std::to_string(r) + " is an equality; its bounds cannot be freed"); return -1; }
      taken[r] = 1;
    }
    const int g[6] = {D->chk_off[k], D->chk_len[k], D->rad_off[k], D->rad_len[k], D->row_off[k], D->row_len[k]};
    std::copy(g, g + 6, geo.begin() + 6 * k);
    rec.insert(rec.end(), ptpl.begin() + g[0], ptpl.begin() + g[0] + g[1]);
    rec.insert(rec.end(), ptpl.begin() + g[2], ptpl.begin() + g[2] + g[3]);
  }
  const size_t B = M.B, ns = rec.size();
  std::vector<double> shapes(B * ns), lb(B * m), ub(B * m);
  for (size_t b = 0; b < B; ++b) {
    std::copy(rec.begin(), rec.end(), shapes.begin() + b * ns);
    std::copy(lbg.begin(), lbg.end(), lb.begin() + b * m);
    std::copy(ubg.begin(), ubg.end(), ub.begin() + b * m);
  }
  bool ok = true;
  const int* d_geo = (const int*)mpc_alloc(q, 4 * geo.size(), geo.data(), &ok);
  double* d_shapes = (double*)mpc_alloc(q, 8 * shapes.size(), shapes.data(), &ok);
  double* d_lbg = (double*)mpc_alloc(q, 8 * lb.size(), lb.data(), &ok);
  double* d_ubg = (double*)mpc_alloc(q, 8 * ub.size(), ub.data(), &ok);
  q->hshapes = (double*)mpc_alloc(q, 8 * shapes.size(), nullptr, &ok);
  q->havoid = (int*)mpc_alloc(q, 4 * B * n_obs, nullptr, &ok);
  if (!ok) { set_err(f + "device allocation/upload failed"); return -1; }
  M.m = m; M.n_shape = (int)ns; M.obs_geo = d_geo; M.lbg = d_lbg; M.ubg = d_ubg;
  M.shapes = d_shapes;                     // (last: a non-null shapes marks the handle attached)
  return 0;
}

int omg_mpc_set_obstacles(omg_mpc* q, const double* shapes, const int32_t* avoid, void* stream_) {
  if (!q) { set_err("omg_mpc_set_obstacles: null argument"); return -1; }
  if (!q->M.shapes) { set_err("omg_mpc_set_obstacles: no obstacles attached (omg_mpc_attach_obstacles)"); return -1; }
  if (!shapes && !avoid) return 0;
  CK(cudaSetDevice(q->h->device));
  OMG_LAUNCH(omg_mpc_set_obstacles_kernel, q->M.B, OMG_MPC_NT, 0, (cudaStream_t)stream_, q->M, shapes, avoid,
             q->h->lbg, q->h->ubg);
  CK(cudaGetLastError());
  return 0;
}

int omg_mpc_set_obstacles_host(omg_mpc* q, const double* shapes, const int32_t* avoid) {
  if (!q) { set_err("omg_mpc_set_obstacles_host: null argument"); return -1; }
  if (!q->M.shapes) { set_err("omg_mpc_set_obstacles_host: no obstacles attached (omg_mpc_attach_obstacles)"); return -1; }
  CK(cudaSetDevice(q->h->device));
  const size_t b = q->M.B;
  if (shapes) CK(cudaMemcpy(q->hshapes, shapes, b * q->M.n_shape * 8, cudaMemcpyHostToDevice));
  if (avoid) CK(cudaMemcpy(q->havoid, avoid, b * q->M.n_obs * 4, cudaMemcpyHostToDevice));
  if (omg_mpc_set_obstacles(q, shapes ? q->hshapes : nullptr, avoid ? q->havoid : nullptr, nullptr)) return -1;
  CK(cudaStreamSynchronize(nullptr));
  return 0;
}

}  // extern "C"
