/* TEST INFRASTRUCTURE - NOT PRODUCT CODE, never loaded by the package.
 *
 * The reference's forward dynamics WITH external forces on the C oracle: oracle/tds_oracle.c is included as it stands (its
 * forward_dynamics drops f_ext, "f_ext = 0 after clear_forces"), and its ABA is restated here with the f_ext term of kinematics.hpp:132,
 * pA = v x* I v - X_world^-1 f_ext.  A link's f_ext is the world spatial force [n + x x f; f] about the world origin, summed over its points
 * (x = the point's world position), mapped into the link frame; for a point on a floating base the same term goes into the base's bias
 * force in the base frame.  Independent of the kernel's common-frame arithmetic.  Bound by tests/emu_wrench.py.
 *   gcc -std=c11 -O2 -fPIC -shared -I<include> -I<oracle> tests/cpp/oracle_wrench.c -o tests/cpp/_oracle_wrench.so -lm */
#include "../../oracle/tds_oracle.c"

/* X^-1 applied to the world force [n; f] about the world origin: [R^T (n - t x f); R^T f] */
static void xf_force_to_local(const Xf* X, const double* n, const double* f, Sv* out) {
  double txf[3], m[3];
  cross3(X->t, f, txf);
  for (int k = 0; k < 3; ++k) m[k] = n[k] - txf[k];
  m3t_v(X->R, m, out->top);
  m3t_v(X->R, f, out->bot);
}

/* qdd [n_qd] of forward_dynamics (forward_dynamics.hpp:11-326) at q, qd, tau [n_tau] with K wrenches W [K][6] = [n; f] (world axes) at the
 * points links[k] (-1: the base) / local[3k..3k+2].  Returns 0, or < 0. */
int tdso_wrench_fd(const double* model, const double* q, const double* qd, const double* tau, const double* gravity, int K, const int* links,
                   const double* local, const double* W, double* qdd) {
  Model M;
  int rc = model_open(model, &M);
  if (rc) return rc;
  State* st = &g_state;
  forward_kinematics(&M, st, q, qd);
  for (int k = 0; k < K; ++k) {   /* kinematics.hpp:132 (links) and :54-61 (the base): - X_world^-1 f_ext */
    const int l = links[k];
    if (l < 0 && !M.floating) continue;   /* the world absorbs a wrench on a fixed base */
    const Xf* X = l >= 0 ? &st->X_world[l] : &st->base_X_world;
    double x[3], xf[3], nw[3];
    m3_v(X->R, local + 3 * k, x);
    for (int c = 0; c < 3; ++c) x[c] += X->t[c];
    cross3(x, W + 6 * k + 3, xf);
    for (int c = 0; c < 3; ++c) nw[c] = W[6 * k + c] + xf[c];
    Sv fl;
    xf_force_to_local(X, nw, W + 6 * k + 3, &fl);
    Sv* pA = l >= 0 ? &st->pA[l] : &st->base_bias_force;
    for (int c = 0; c < 3; ++c) { pA->top[c] -= fl.top[c]; pA->bot[c] -= fl.bot[c]; }
  }
  /* the rest of forward_dynamics as oracle/tds_oracle.c states it */
  for (int i = M.n_links - 1; i >= 0; --i) { /* forward_dynamics.hpp:50-216 */
    const double* l = LNK(&M, i);
    int parent = (int)l[TDSM_L_PARENT];
    int jt = (int)l[TDSM_L_JTYPE];
    abi_mul(&st->abi[i], &st->S[i], &st->U[i]);
    st->D[i] = sv_dot(&st->S[i], &st->U[i]);
    double tau_val = 0.0;
    if (jt != TDSJ_FIXED) {
      int qdi = (int)l[TDSM_L_QDIDX];
      tau_val = tau ? tau[qdi - (M.floating ? 6 : 0)] : 0.0;
      tau_val -= l[TDSM_L_STIFFNESS] * q[(int)l[TDSM_L_QIDX]];
      tau_val -= l[TDSM_L_DAMPING] * qd[qdi];
    }
    st->u[i] = tau_val - sv_dot(&st->S[i], &st->pA[i]);
    double invD = (jt == TDSJ_FIXED) ? 0.0 : 1.0 / st->D[i];
    Abi Ia = st->abi[i];
    Sv UinvD;
    for (int k = 0; k < 3; ++k) { UinvD.top[k] = st->U[i].top[k] * invD; UinvD.bot[k] = st->U[i].bot[k] * invD; }
    for (int r = 0; r < 3; ++r)
      for (int cc = 0; cc < 3; ++cc) {
        Ia.I[r * 3 + cc] -= st->U[i].top[r] * UinvD.top[cc];
        Ia.H[r * 3 + cc] -= st->U[i].top[r] * UinvD.bot[cc];
        Ia.M[r * 3 + cc] -= st->U[i].bot[r] * UinvD.bot[cc];
      }
    Sv Ia_c, pa, dpA;
    abi_mul(&Ia, &st->c[i], &Ia_c);
    double uD = st->u[i] * invD;
    for (int k = 0; k < 3; ++k) {
      pa.top[k] = st->pA[i].top[k] + Ia_c.top[k] + st->U[i].top[k] * uD;
      pa.bot[k] = st->pA[i].bot[k] + Ia_c.bot[k] + st->U[i].bot[k] * uD;
    }
    xf_apply_force(&st->X_parent[i], &pa, &dpA);
    Abi dI;
    xt_abi_x(&st->X_parent[i], &Ia, &dI);
    if (parent >= 0) {
      for (int k = 0; k < 3; ++k) { st->pA[parent].top[k] += dpA.top[k]; st->pA[parent].bot[k] += dpA.bot[k]; }
      abi_add(&st->abi[parent], &dI);
    } else if (M.floating) {
      for (int k = 0; k < 3; ++k) { st->base_bias_force.top[k] += dpA.top[k]; st->base_bias_force.bot[k] += dpA.bot[k]; }
      abi_add(&st->base_abi, &dI);
    }
  }
  if (M.floating) {
    Sv r;
    abi_inv_mul(&st->base_abi, &st->base_bias_force, &r);
    for (int k = 0; k < 3; ++k) { st->base_acc.top[k] = -r.top[k]; st->base_acc.bot[k] = -r.bot[k]; }
  } else {
    for (int k = 0; k < 3; ++k) { st->base_acc.top[k] = 0.0; st->base_acc.bot[k] = -gravity[k]; }
  }
  for (int i = 0; i < M.n_links; ++i) {
    const double* l = LNK(&M, i);
    int parent = (int)l[TDSM_L_PARENT];
    int jt = (int)l[TDSM_L_JTYPE];
    const Sv* ap = parent >= 0 ? &st->a[parent] : &st->base_acc;
    Sv xa;
    xf_apply_motion(&st->X_parent[i], ap, &xa);
    for (int k = 0; k < 3; ++k) { st->a[i].top[k] = xa.top[k] + st->c[i].top[k]; st->a[i].bot[k] = xa.bot[k] + st->c[i].bot[k]; }
    if (jt != TDSJ_FIXED) {
      double invD = 1.0 / st->D[i];
      double qddv = invD * (st->u[i] - sv_dot(&st->U[i], &st->a[i]));
      qdd[(int)l[TDSM_L_QDIDX]] = qddv;
      for (int k = 0; k < 3; ++k) { st->a[i].top[k] += st->S[i].top[k] * qddv; st->a[i].bot[k] += st->S[i].bot[k] * qddv; }
    }
  }
  if (M.floating) {
    for (int k = 0; k < 3; ++k) { st->base_acc.bot[k] += gravity[k]; }
    for (int k = 0; k < 3; ++k) { qdd[k] = st->base_acc.top[k]; qdd[3 + k] = st->base_acc.bot[k]; }
  }
  return 0;
}
