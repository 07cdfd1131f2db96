// Newton solver (primal) of the batched mj_step path for ONE environment, cooperative lanes.
//
// Replaces (reference file:line) src/engine/engine_solver.c: mjPrimalContext :979-1092,
// PrimalUpdateConstraint :1370-1404, PrimalUpdateGrad/Mgrad :1407-1448, PrimalPrepare :1451-1524,
// frictionCost/frictionCostDif :1536-1571, PrimalEval :1675-1822, updateBracket :1826-1853,
// PrimalSearch :1856-2052, MakeHessian (dense) :2133-2141, FactorizeHessian (dense) :2196-2208,
// HessianIncremental :2285-2340, mj_solPrimal (Newton branch) :2344-2563; and the dense Cholesky
// kernels of src/engine/engine_util_solve.c: mju_cholFactor :33-70, mju_cholSolve :74-100,
// mju_cholUpdate :104-147; mju_sqrMatTD_impl (engine_util_blas.c), mju_addToSymSparse and
// mju_mulSymVecSparse (engine_util_sparse.c).
//
// Scope: dense Jacobian (any nv), pyramidal cones, no equality rows, one kinematic tree (so the
// constraint island, when islands are enabled, is the whole system and its dof / row order is the
// global one: engine_island.c:455-650; only the cost scale differs, 1/trace(M) instead of
// 1/(meaninertia*nv), engine_solver.c:2383-2394).
//
// Parallel structure: matrix-shaped work is spread over the lanes element by element (Hessian
// elements, Cholesky column updates, Jacobian rows), every element keeping the reference's
// accumulation order.  The scalar control flow of the line search and all order-sensitive scalar
// sums are evaluated by every lane redundantly on identical data, so decisions are warp-uniform
// without broadcasts.  The two triangular solves are inherently serial chains (lane 0).
#pragma once
#include "mjb_constraint.h"

namespace mjb {

struct LsPoint { double alpha, cost, d0, d1; };

// the sub-problem one primal solve works on: all rows and dofs (monolithic), or the rows and dofs of one
// constraint island in island order (engine_solver.c PrimalPointers/PrimalAllocate :1095-1366: the
// reference gathers island-local copies iacc, ifrc_*, iM, iefc_J; here the global arrays are indexed
// through the island maps, which performs the same arithmetic on the same operands in the same order)
// ISL = false is the identity view (monolithic problem): the maps fold away at compile time
template <bool ISL>
struct IslView {
  const int* rows; int nrow;      // island row c -> global efc row
  const int* dofs; int ndof;      // island dof k -> global dof
  const int* dof2idof; int base;  // global dof -> island dof = dof2idof[dof] - base
  MJB_HD int row(int c) const { return ISL ? rows[c] : c; }
  MJB_HD int dof(int k) const { return ISL ? dofs[k] : k; }
  MJB_HD int loc(int dof_) const { return ISL ? dof2idof[dof_] - base : dof_; }
};

template <bool ISL>
struct NewtonCtx {
  IslView<ISL> v;
  int nv, nefc, ne, nf;           // nv: global dof count (row pitch of J); nefc: global; rows [0,ne) equality,
                                  // [ne,nf) friction (nf = END of the friction rows)
  FD J, Jaref, Jv, quad, Dq, Ma, Mv, grad, Mgrad, search, cholupd, L;   // Ma..cholupd, L: island-local
  FD efcD, efcR, floss, qfs, qas, qacc;
  FI state, oldstate;
  double quadGauss[3];
  double scale, cost;
  int lsiter;
};

// Huber cost of a friction row and its difference between two points
MJB_HD double friction_cost(double x, double f, double Rf, double D) {
  if (-Rf < x && x < Rf) return 0.5 * D * x * x;
  else if (x <= -Rf) return f * (-0.5 * Rf - x);
  else return f * (-0.5 * Rf + x);
}
MJB_HD double friction_cost_dif(double start, double x, double f, double Rf, double D) {
  const int s0 = (-Rf < start && start < Rf) ? 0 : (start <= -Rf ? -1 : 1);
  const int s1 = (-Rf < x && x < Rf) ? 0 : (x <= -Rf ? -1 : 1);
  if (s0 == 0 && s1 == 0) return 0.5 * D * (x - start) * (x + start);
  if (s0 == -1 && s1 == -1) return f * (start - x);
  if (s0 == 1 && s1 == 1) return f * (x - start);
  return friction_cost(x, f, Rf, D) - friction_cost(start, f, Rf, D);
}

// res = M * vec on the view's dofs (vectors island-local): mju_mulSymVecSparse order per output dof —
// diagonal term, own-row off-diagonals from the last column to the first, descendant rows ascending
template <bool ISL>
MJB_HD void mul_M_view(const Env& d, const IslView<ISL>& v, FD res, FD vec) {
  const DModel& m = d.m;
  FD M = d.M();
  MJB_PFOR(k, v.ndof) {
    const int i = v.dof(k);
    const int adr = m.M_rowadr[i], nnz = m.M_rownnz[i];
    double s = M[adr + nnz - 1] * vec[k];
    for (int a = nnz - 2; a >= 0; a--) s += M[adr + a] * vec[v.loc(m.M_colind[adr + a])];
    const int a0 = m.mt_adr[i], an = m.mt_adr[i + 1] - a0;
    for (int c = an - 1; c >= 0; c--) s += M[m.mt_qadr[a0 + c]] * vec[v.loc(m.mt_dof[a0 + c])];
    res[k] = s;
  }
  MJB_PSYNC();
}

// res[row] = J(row, view dofs) . vec   (mju_mulMatVec on the island block)
template <bool ISL>
MJB_HD void mul_jac_view(const Env& d, const NewtonCtx<ISL>& c, FD res, FD vec) {
  const IslView<ISL>& v = c.v;
  MJB_PFOR(cc, v.nrow) {
    const int i = v.row(cc);
    res[i] = dot_ref(v.ndof, [&](int k) { return c.J[(long)i * c.nv + v.dof(k)]; }, [&](int k) { return vec[k]; });
  }
  MJB_PSYNC();
}

// x = M^-1 x for an island-local vector: embedded in a global vector (zeros elsewhere; trees do not
// couple in L'DL, so the island's dofs see exactly the operations of the block solve)
template <bool ISL>
MJB_HD void solve_M_view(const Env& d, const IslView<ISL>& v, FD x) {
  if (!ISL) { solve_LD(d, x, d.qLD(), d.qLDiagInv()); return; }
  FD g = d.scr_nv() + 2 * d.m.sz.nv;
  MJB_PFOR(i, d.m.sz.nv) g[i] = 0;
  MJB_PSYNC();
  MJB_PFOR(k, v.ndof) g[v.dof(k)] = x[k];
  MJB_PSYNC();
  solve_LD(d, g, d.qLD(), d.qLDiagInv());
  MJB_PFOR(k, v.ndof) x[k] = g[v.dof(k)];
  MJB_PSYNC();
}

// efc_force / efc_state / cost from Jaref (mj_constraintUpdate_impl on the view's rows),
// qfrc_constraint = J' force on the view's dofs, plus the Gauss term
template <bool ISL>
MJB_HD void newton_update_constraint(const Env& d, NewtonCtx<ISL>& c) {
  const IslView<ISL>& v = c.v;
  FD force = d.efc_force(), qfc = d.qfrc_constraint();
  MJB_PFOR(cc, v.nrow) {
    const int i = v.row(cc);
    const double jar = c.Jaref[i];
    double f = -c.efcD[i] * jar;
    int st;
    if (i < c.ne) st = STATE_QUADRATIC;
    else if (i < c.nf) {
      if (jar <= -c.efcR[i] * c.floss[i]) { f = c.floss[i]; st = STATE_LINEARNEG; }
      else if (jar >= c.efcR[i] * c.floss[i]) { f = -c.floss[i]; st = STATE_LINEARPOS; }
      else st = STATE_QUADRATIC;
    } else if (jar >= 0) { f = 0; st = STATE_SATISFIED; }
    else st = STATE_QUADRATIC;
    force[i] = f; c.state[i] = st;
  }
  MJB_PSYNC();
  double s = 0;
  for (int cc = 0; cc < v.nrow; cc++) {
    const int i = v.row(cc), st = c.state[i];
    const double jar = c.Jaref[i];
    if (st == STATE_LINEARNEG) s += -0.5 * c.efcR[i] * c.floss[i] * c.floss[i] - c.floss[i] * jar;
    else if (st == STATE_LINEARPOS) s += -0.5 * c.efcR[i] * c.floss[i] * c.floss[i] + c.floss[i] * jar;
    else if (st == STATE_QUADRATIC) s += 0.5 * c.efcD[i] * jar * jar;
  }
  MJB_PFOR(k, v.ndof) {
    const int dof = v.dof(k);
    double q = 0;
    for (int cc = 0; cc < v.nrow; cc++) {
      const int i = v.row(cc);
      const double f = force[i];
      if (f != 0) q += c.J[(long)i * c.nv + dof] * f;
    }
    qfc[dof] = q;
  }
  MJB_PSYNC();
  double gauss = 0;
  for (int k = 0; k < v.ndof; k++) { const int dof = v.dof(k); gauss += 0.5 * (c.Ma[k] - c.qfs[dof]) * (c.qacc[dof] - c.qas[dof]); }
  c.quadGauss[0] = gauss;
  s += gauss;
  c.cost = s;
}

template <bool ISL>
MJB_HD void newton_update_grad(const Env& d, NewtonCtx<ISL>& c) {
  FD qfc = d.qfrc_constraint();
  MJB_PFOR(k, c.v.ndof) { const int dof = c.v.dof(k); c.grad[k] = c.Ma[k] - c.qfs[dof] - qfc[dof]; }
  MJB_PSYNC();
}

// in-place dense Cholesky of the lower triangle; returns the rank (uniform)
MJB_HD int chol_factor(const Env& d, FD mat, int n, double mindiag) {
  int rank = n;
  for (int j = 0; j < n; j++) {
    double tmp = mat[j * (n + 1)];
    if (j) tmp -= dot_ref(j, [&](int k) { return mat[j * n + k]; }, [&](int k) { return mat[j * n + k]; });
    const bool deficient = tmp < mindiag;
    if (deficient) { tmp = mindiag; rank--; }
    const double diag = sqrt(tmp);
    MJB_PSYNC();
    MJB_LANE0 mat[j * (n + 1)] = diag;
    if (deficient) {
      MJB_PFOR(i_, n - 1 - j) mat[(j + 1 + i_) * n + j] = 0;
    } else {
      const double inv = 1 / diag;
      MJB_PFOR(i_, n - 1 - j) {
        const int i = j + 1 + i_;
        mat[i * n + j] = (mat[i * n + j] - dot_ref(j, [&](int k) { return mat[i * n + k]; },
                                                   [&](int k) { return mat[j * n + k]; })) * inv;
      }
    }
    MJB_PSYNC();
  }
  return rank;
}

// res = (L L')^-1 vec: forward then backward substitution, serial chains
MJB_HD void chol_solve(const Env& d, FD res, FD mat, FD vec, int n) {
  MJB_LANE0 {
    for (int i = 0; i < n; i++) res[i] = vec[i];
    for (int i = 0; i < n; i++) {
      if (i) res[i] -= dot_ref(i, [&](int k) { return mat[i * n + k]; }, [&](int k) { return res[k]; });
      res[i] /= mat[i * (n + 1)];
    }
    for (int i = n - 1; i >= 0; i--) {
      double r = res[i];
      for (int j = i + 1; j < n; j++) r -= mat[j * n + i] * res[j];
      res[i] = r / mat[i * (n + 1)];
    }
  }
  MJB_PSYNC();
}

// rank-one update (plus) or downdate of the factor with x (destroyed); returns the rank (uniform)
MJB_HD int chol_update(const Env& d, FD mat, FD x, int n, bool plus) {
  int rank = n;
  for (int k = 0; k < n; k++) {
    const double xk = x[k];
    if (xk != 0) {
      const double Lkk = mat[k * (n + 1)];
      double tmp = Lkk * Lkk + (plus ? xk * xk : -xk * xk);
      if (tmp < kMinVal) { tmp = kMinVal; rank--; }
      const double r = sqrt(tmp);
      const double cc = r / Lkk;
      const double cinv = 1 / cc;
      const double s = xk / Lkk;
      MJB_PSYNC();
      MJB_LANE0 mat[k * (n + 1)] = r;
      MJB_PFOR(i_, n - 1 - k) {
        const int i = k + 1 + i_;
        double mv = mat[i * n + k];
        mv = plus ? (mv + s * x[i]) * cinv : (mv - s * x[i]) * cinv;
        mat[i * n + k] = mv;
        x[i] = cc * x[i] - s * mv;
      }
      MJB_PSYNC();
    }
  }
  return rank;
}

// L <- lower triangle of H = M + J' diag(Dq) J on the view (island-local n x n), then its Cholesky factor
template <bool ISL>
MJB_HD void newton_factorize(const Env& d, NewtonCtx<ISL>& c, bool recompute) {
  const DModel& m = d.m;
  const IslView<ISL>& v = c.v;
  const int n = v.ndof, nv = c.nv;
  if (recompute) {
    MJB_PFOR(cc, v.nrow) { const int i = v.row(cc); c.Dq[i] = (c.state[i] == STATE_QUADRATIC) ? c.efcD[i] : 0.0; }
    MJB_PSYNC();
    MJB_PFOR(e, n * n) {
      const int a = e / n, b = e - a * n;
      double s = 0;
      if (b <= a) {
        const int da = v.dof(a), db = v.dof(b);
        for (int cc = 0; cc < v.nrow; cc++) {
          const int j = v.row(cc);
          const double dj = c.Dq[j];
          if (dj != 0) {
            const double t = c.J[(long)j * nv + da];
            if (t != 0) s += c.J[(long)j * nv + db] * (t * dj);
          }
        }
      }
      c.L[e] = s;
    }
    MJB_PSYNC();
    FD M = d.M();
    MJB_PFOR(a, n) {
      const int i = v.dof(a);
      const int adr = m.M_rowadr[i], nnz = m.M_rownnz[i];
      for (int q = 0; q < nnz; q++) c.L[a * n + v.loc(m.M_colind[adr + q])] += M[adr + q];
    }
    MJB_PSYNC();
  }
  chol_factor(d, c.L, n, kMinVal);
}

template <bool ISL>
MJB_HD void newton_update_mgrad(const Env& d, NewtonCtx<ISL>& c) { chol_solve(d, c.Mgrad, c.L, c.grad, c.v.ndof); }

// rank-one updates of the factor for the rows whose QUADRATIC membership changed
template <bool ISL>
MJB_HD void newton_hessian_incremental(const Env& d, NewtonCtx<ISL>& c) {
  const IslView<ISL>& v = c.v;
  const int n = v.ndof;
  for (int cc = 0; cc < v.nrow; cc++) {
    const int i = v.row(cc);
    const bool was = c.oldstate[i] == STATE_QUADRATIC, is = c.state[i] == STATE_QUADRATIC;
    if (was == is) continue;
    const double sq = sqrt(c.efcD[i]);
    MJB_PFOR(k, n) c.cholupd[k] = c.J[(long)i * c.nv + v.dof(k)] * sq;
    MJB_PSYNC();
    const int rank = chol_update(d, c.L, c.cholupd, n, is);
    if (rank < n) {
      newton_factorize(d, c, true);
      return;
    }
  }
}

// line-search objective and its first two derivatives at p.alpha (cost relative to alpha = 0)
template <bool ISL>
MJB_HD void newton_eval(NewtonCtx<ISL>& c, LsPoint& p) {
  const double alpha = p.alpha;
  double cost = 0, d0 = 0, d1 = 0;
  double q0 = 0, q1 = c.quadGauss[1], q2 = c.quadGauss[2];
  for (int cc = 0; cc < c.v.nrow; cc++) {
    const int i = c.v.row(cc);
    if (i < c.ne) {   // equality: shifted quadratic (quad[0] dropped)
      q1 += c.quad[3 * i + 1];
      q2 += c.quad[3 * i + 2];
      continue;
    }
    if (i < c.nf) {
      const double start = c.Jaref[i], dir = c.Jv[i];
      const double x = start + alpha * dir;
      const double f = c.floss[i], D = c.efcD[i];
      const double Rf = c.efcR[i] * f;
      cost += friction_cost_dif(start, x, f, Rf, D);
      if (-Rf < x && x < Rf) { d0 += D * x * dir; d1 += D * dir * dir; }
      else if (x <= -Rf) d0 += -f * dir;
      else d0 += f * dir;
      continue;
    }
    const double start = c.Jaref[i];
    const double x = start + alpha * c.Jv[i];
    const double cost0 = start < 0 ? c.quad[3 * i] : 0;
    if (x < 0) {
      q0 += c.quad[3 * i] - cost0;
      q1 += c.quad[3 * i + 1];
      q2 += c.quad[3 * i + 2];
    } else {
      cost -= cost0;
    }
  }
  cost += alpha * alpha * q2 + alpha * q1 + q0;
  d0 += 2 * alpha * q2 + q1;
  d1 += 2 * q2;
  if (d1 <= 0) d1 = kMinVal;
  p.cost = cost; p.d0 = d0; p.d1 = d1;
  c.lsiter++;
}

template <bool ISL>
MJB_HD int newton_update_bracket(NewtonCtx<ISL>& c, LsPoint& p, const LsPoint* cand, LsPoint& pnext) {
  int flag = 0;
  for (int i = 0; i < 3; i++) {
    if (p.d0 < 0 && cand[i].d0 < 0 && p.d0 < cand[i].d0) { p = cand[i]; flag = 1; }
    else if (p.d0 > 0 && cand[i].d0 > 0 && p.d0 > cand[i].d0) { p = cand[i]; flag = 2; }
  }
  if (flag) {
    pnext.alpha = p.alpha - p.d0 / p.d1;
    newton_eval(c, pnext);
  }
  return flag;
}

// exact line search along `search`; returns the step and the cost improvement
template <bool ISL>
MJB_HD double newton_search(const Env& d, NewtonCtx<ISL>& c, double tolerance, int ls_iterations, double& improvement) {
  const IslView<ISL>& v = c.v;
  const int n = v.ndof;
  c.lsiter = 0;
  improvement = 0;
  const double snorm = sqrt(dot_ref(n, [&](int k) { return c.search[k]; }, [&](int k) { return c.search[k]; }));
  if (snorm < kMinVal) return 0;
  const double gtol = tolerance * snorm / c.scale;

  mul_M_view(d, v, c.Mv, c.search);
  mul_jac_view(d, c, c.Jv, c.search);

  // quadratic polynomials (PrimalPrepare)
  c.quadGauss[1] = dot_ref(n, [&](int k) { return c.search[k]; }, [&](int k) { return c.Ma[k]; }) -
                   dot_ref(n, [&](int k) { return c.qfs[v.dof(k)]; }, [&](int k) { return c.search[k]; });
  c.quadGauss[2] = 0.5 * dot_ref(n, [&](int k) { return c.search[k]; }, [&](int k) { return c.Mv[k]; });
  MJB_PFOR(cc, v.nrow) {
    const int i = v.row(cc);
    const double D = c.efcD[i], ja = c.Jaref[i], jv = c.Jv[i];
    const double DJ0 = D * ja;
    c.quad[3 * i] = ja * DJ0 * 0.5;
    c.quad[3 * i + 1] = jv * DJ0;
    c.quad[3 * i + 2] = jv * D * jv * 0.5;
  }
  MJB_PSYNC();

  LsPoint p0, p1, p2, pmid, p1next, p2next;
  p0.alpha = 0;
  newton_eval(c, p0);
  p1.alpha = p0.alpha - p0.d0 / p0.d1;
  newton_eval(c, p1);
  if (fabs(p1.d0) < gtol && (p1.alpha == 0 || p1.cost < 0)) {
    improvement = -p1.cost;
    return p1.alpha;
  }
  const int dir = (p1.d0 < 0 ? +1 : -1);

  // one-sided search
  p2 = p0;
  while (p1.d0 * dir <= -gtol && c.lsiter < ls_iterations) {
    p2 = p1;
    p1.alpha -= p1.d0 / p1.d1;
    newton_eval(c, p1);
    if (fabs(p1.d0) < gtol && p1.cost < 0) {
      improvement = -p1.cost;
      return p1.alpha;
    }
  }
  if (c.lsiter >= ls_iterations) {
    improvement = -p1.cost;
    return p1.alpha;
  }

  // bracketed search
  p2next = p1;
  p1next.alpha = p1.alpha - p1.d0 / p1.d1;
  newton_eval(c, p1next);
  while (c.lsiter < ls_iterations) {
    pmid.alpha = 0.5 * (p1.alpha + p2.alpha);
    newton_eval(c, pmid);
    LsPoint cand[3] = {p1next, p2next, pmid};
    double bestcost = 0;
    int bestind = -1;
    for (int i = 0; i < 3; i++) {
      if (fabs(cand[i].d0) < gtol && (bestind == -1 || cand[i].cost < bestcost)) {
        bestcost = cand[i].cost;
        bestind = i;
      }
    }
    if (bestind >= 0) {
      improvement = -cand[bestind].cost;
      return cand[bestind].alpha;
    }
    const int b1 = newton_update_bracket(c, p1, cand, p1next);
    const int b2 = newton_update_bracket(c, p2, cand, p2next);
    if (!b1 && !b2) {
      improvement = -pmid.cost;
      return pmid.alpha;
    }
  }
  if (p1.cost <= p2.cost && p1.cost < 0) { improvement = -p1.cost; return p1.alpha; }
  else if (p2.cost <= p1.cost && p2.cost < 0) { improvement = -p2.cost; return p2.alpha; }
  return 0;
}

// Newton (newton = true) or conjugate gradient (mj_solCG: M-preconditioned, Hager-Zhang direction
// update, engine_solver.c:2489-2518) on the primal problem of one view; returns the iteration count
template <bool ISL>
MJB_HD int solve_primal_view(const Env& d, bool newton, const IslView<ISL>& view, bool island_scale) {
  const DModel& m = d.m;
  const int nv = m.sz.nv, njmax = m.sz.njmax;
  NewtonCtx<ISL> c;
  c.v = view;
  const IslView<ISL>& v = c.v;
  const int n = v.ndof;
  c.nv = nv; c.nefc = d.nefc()[0]; c.ne = d.ne()[0]; c.nf = c.ne + d.nf()[0];
  c.J = d.efc_J();
  FD se = d.nwt_efc(), sv = d.nwt_nv();
  c.Jaref = se; c.Jv = se + njmax; c.quad = se + 2 * (long)njmax; c.Dq = se + 5 * (long)njmax;
  c.Ma = sv; c.Mv = sv + nv; c.grad = sv + 2 * nv; c.Mgrad = sv + 3 * nv; c.search = sv + 4 * nv; c.cholupd = sv + 5 * nv;
  FD gradold = d.scr_nv(), Mgradold = d.scr_nv() + nv;   // CG only
  c.L = d.nwt_L();
  c.efcD = d.efc_D(); c.efcR = d.efc_R(); c.floss = d.efc_frictionloss();
  c.qfs = d.qfrc_smooth(); c.qas = d.qacc_smooth(); c.qacc = d.qacc();
  c.state = d.efc_state(); c.oldstate = d.nwt_state();
  const double tol = m.opt.tolerance;

  // Ma = M qacc (island-local), Jaref = J qacc - aref
  {
    FD qa = c.search;   // island-local copy of qacc (search is free until the first direction)
    MJB_PFOR(k, n) qa[k] = c.qacc[v.dof(k)];
    MJB_PSYNC();
    mul_M_view(d, v, c.Ma, qa);
    mul_jac_view(d, c, c.Jaref, qa);
    FD aref = d.efc_aref();
    MJB_PFOR(cc, v.nrow) { const int i = v.row(cc); c.Jaref[i] -= aref[i]; }
    MJB_PSYNC();
  }
  newton_update_constraint(d, c);
  newton_update_grad(d, c);

  // cost scale: the island's (trace of its M block), the global one when islands are not in use
  if (island_scale) {
    FD M = d.M();
    double tr = 0;
    for (int k = 0; k < n; k++) { const int i = v.dof(k); tr += M[m.M_rowadr[i] + m.M_rownnz[i] - 1]; }
    c.scale = 1 / tr;
  } else {
    c.scale = 1 / (m.opt.meaninertia * (nv > 1 ? nv : 1));
  }
  const double scale = c.scale;

  // convergence certificate with the M-preconditioned gradient
  MJB_PFOR(k, n) c.Mgrad[k] = c.grad[k];
  MJB_PSYNC();
  solve_M_view(d, v, c.Mgrad);
  auto grad_dot_mgrad = [&]() { return dot_ref(n, [&](int k) { return c.grad[k]; }, [&](int k) { return c.Mgrad[k]; }); };
  auto grad_norm = [&]() { return sqrt(dot_ref(n, [&](int k) { return c.grad[k]; }, [&](int k) { return c.grad[k]; })); };
  const bool flg_gap = dmax(0.0, 0.5 * scale * grad_dot_mgrad()) < tol;
  const bool flg_gradient = scale * grad_norm() < tol;
  bool done = flg_gap && (!newton || flg_gradient);
  MJB_PSYNC();

  if (!done && newton) {
    newton_factorize(d, c, true);
    newton_update_mgrad(d, c);
    done = flg_gradient && dmax(0.0, 0.5 * scale * grad_dot_mgrad()) < tol;
  }
  if (!done) {
    MJB_PFOR(k, n) c.search[k] = c.Mgrad[k] * -1;
    MJB_PSYNC();
  }

  int iter = 0;
  const int maxiter = m.opt.iterations;
  while (!done && iter < maxiter) {
    double ls_improvement;
    const double alpha = newton_search(d, c, tol * m.opt.ls_tolerance, m.opt.ls_iterations, ls_improvement);
    if (alpha == 0) break;
    MJB_PSYNC();
    MJB_PFOR(k, n) { c.qacc[v.dof(k)] += c.search[k] * alpha; c.Ma[k] += c.Mv[k] * alpha; }
    MJB_PFOR(cc, v.nrow) { const int i = v.row(cc); c.Jaref[i] += c.Jv[i] * alpha; c.oldstate[i] = c.state[i]; }
    if (!newton) { MJB_PFOR(k, n) { gradold[k] = c.grad[k]; Mgradold[k] = c.Mgrad[k]; } }
    MJB_PSYNC();
    newton_update_constraint(d, c);
    if (newton) newton_hessian_incremental(d, c);
    newton_update_grad(d, c);
    if (newton) {
      newton_update_mgrad(d, c);
    } else {
      MJB_PFOR(k, n) c.Mgrad[k] = c.grad[k];
      MJB_PSYNC();
      solve_M_view(d, v, c.Mgrad);
    }
    const double improvement = scale * ls_improvement;
    const double gradient = scale * grad_norm();
    const double decrement = newton ? dmax(0.0, 0.5 * scale * grad_dot_mgrad()) : 0.0;
    iter++;
    if ((improvement > 0 && improvement < tol) || gradient < tol || (newton && decrement < tol)) break;
    MJB_PSYNC();
    if (newton) {
      MJB_PFOR(k, n) c.search[k] = c.Mgrad[k] * -1;
    } else {
      // Hager-Zhang: every lane evaluates the same dot products (uniform beta)
      auto dotf = [&](auto a, auto b) { return dot_ref(n, a, b); };
      auto S = [&](int k) { return c.search[k]; };
      auto Y = [&](int k) { return c.grad[k] - gradold[k]; };
      auto MY = [&](int k) { return c.Mgrad[k] - Mgradold[k]; };
      auto G = [&](int k) { return c.grad[k]; };
      auto MG = [&](int k) { return c.Mgrad[k]; };
      double beta;
      const double d_dot_y = dotf(S, Y);
      if (d_dot_y < kMinVal) {
        beta = 0;
      } else {
        const double y_dot_My = dotf(Y, MY), y_dot_Mgrad = dotf(Y, MG), d_dot_grad = dotf(S, G);
        const double beta_hz = (y_dot_Mgrad - 2 * (y_dot_My / d_dot_y) * d_dot_grad) / d_dot_y;
        const double d_norm = sqrt(dotf(S, S)), g_norm = sqrt(dotf(G, G));
        const double eta_k = -1.0 / dmax(kMinVal, d_norm * dmin(0.01, g_norm));
        beta = dmax(eta_k, beta_hz);
      }
      MJB_PSYNC();
      MJB_PFOR(k, n) c.search[k] = -c.Mgrad[k] + beta * c.search[k];
    }
    MJB_PSYNC();
  }
  MJB_PSYNC();
  return iter;
}

// mj_fwdConstraint's dispatch (engine_forward.c:1187-1226): one solve per constraint island when islands
// are in use, the monolithic problem otherwise.  Dofs outside every island keep qacc = qacc_smooth
// (warmstart, engine_forward.c:1121-1128).
MJB_HD void solve_primal(const Env& d, bool newton) {
  const DModel& m = d.m;
  const int nv = m.sz.nv, nefc = d.nefc()[0];
  if (!nefc) return;
  FI niter = d.solver_niter();
  if (use_islands(d)) {
    const int nisland = d.nisland()[0];
    const int* eadr = d.island_iefcadr().p;
    const int* dadr = d.island_idofadr().p;
    for (int k = 0; k < nisland; k++) {
      IslView<true> v{d.map_iefc2efc().p + eadr[k], eadr[k + 1] - eadr[k], d.map_idof2dof().p + dadr[k], dadr[k + 1] - dadr[k],
                      d.map_dof2idof().p, dadr[k]};
      const int iter = solve_primal_view<true>(d, newton, v, true);
      MJB_LANE0 if (k < NISLAND) niter[k] += iter;
      MJB_PSYNC();
    }
  } else {
    IslView<false> v{nullptr, nefc, nullptr, nv, nullptr, 0};
    // a single tree with islands enabled is one island: same problem, island cost scale
    const int iter = solve_primal_view<false>(d, newton, v, !(m.opt.disableflags & DSBL_ISLAND));
    MJB_LANE0 niter[0] += iter;
    MJB_PSYNC();
  }
}

}  // namespace mjb
