/* TEST INFRASTRUCTURE - NOT PRODUCT CODE, never loaded by the package.
 *
 * Inverse dynamics (the recursive Newton-Euler algorithm) restated IN LINK FRAMES on the C oracle: oracle/tds_oracle.c is included as it
 * stands, its static forward_kinematics gives every link's X_parent, S, v, c = v x vJ, rigid inertia and pA = v x* (I v); then the
 * accelerations root to leaf (a_i = X_i a_parent + S_i qdd_i + c_i), f_i = I_i a_i + pA_i, and the forces leaf to root with
 * xf_apply_force.  Independent of the kernel's common-frame arithmetic.  Bound by tests/emu_invdyn.py.
 *   gcc -std=c11 -O2 -fPIC -shared -I<include> -I<oracle> tests/cpp/oracle_invdyn.c -o tests/cpp/_oracle_invdyn.so -lm */
#include "../../oracle/tds_oracle.c"

/* tau [n_qd] at q, qd, qdd (NULL: zero) under gravity[3]: fixed base: joint forces including stiffness q + damping qd; floating base:
 * rows 0..5 the wrench on the base in the base frame [moment; force], qdd[0:6] the base-frame spatial acceleration, gravity rotated into
 * the base frame.  Returns 0, or < 0. */
int tdso_inverse_dynamics(const double* model, const double* q, const double* qd, const double* qdd, const double* gravity, double* tau) {
  static Sv a[MAXL], f[MAXL];
  Model M;
  int rc = model_open(model, &M);
  if (rc) return rc;
  State* st = &g_state;
  forward_kinematics(&M, st, q, qd);
  Sv ab, fb;
  memset(&fb, 0, sizeof fb);
  if (M.floating) {
    double gb[3];
    m3t_v(st->base_X_world.R, gravity, gb);
    for (int k = 0; k < 3; ++k) { ab.top[k] = qdd ? qdd[k] : 0.0; ab.bot[k] = (qdd ? qdd[3 + k] : 0.0) - gb[k]; }
  } else {
    for (int k = 0; k < 3; ++k) { ab.top[k] = 0.0; ab.bot[k] = -gravity[k]; }
  }
  for (int i = 0; i < M.n_links; ++i) {
    const double* l = LNK(&M, i);
    const int parent = (int)l[TDSM_L_PARENT];
    Sv xa, Ia;
    xf_apply_motion(&st->X_parent[i], parent >= 0 ? &a[parent] : &ab, &xa);
    const double qddv = ((int)l[TDSM_L_JTYPE] == TDSJ_FIXED || !qdd) ? 0.0 : qdd[(int)l[TDSM_L_QDIDX]];
    for (int k = 0; k < 3; ++k) {
      a[i].top[k] = xa.top[k] + st->c[i].top[k] + st->S[i].top[k] * qddv;
      a[i].bot[k] = xa.bot[k] + st->c[i].bot[k] + st->S[i].bot[k] * qddv;
    }
    abi_mul(&st->abi[i], &a[i], &Ia);
    for (int k = 0; k < 3; ++k) { f[i].top[k] = Ia.top[k] + st->pA[i].top[k]; f[i].bot[k] = Ia.bot[k] + st->pA[i].bot[k]; }
  }
  memset(tau, 0, sizeof(double) * M.n_qd);
  for (int i = M.n_links - 1; i >= 0; --i) {
    const double* l = LNK(&M, i);
    const int parent = (int)l[TDSM_L_PARENT];
    if ((int)l[TDSM_L_JTYPE] != TDSJ_FIXED) {
      const int qdi = (int)l[TDSM_L_QDIDX];
      tau[qdi] = sv_dot(&st->S[i], &f[i]) + l[TDSM_L_STIFFNESS] * q[(int)l[TDSM_L_QIDX]] + l[TDSM_L_DAMPING] * (qd ? qd[qdi] : 0.0);
    }
    Sv fp;
    xf_apply_force(&st->X_parent[i], &f[i], &fp);
    Sv* to = parent >= 0 ? &f[parent] : (M.floating ? &fb : NULL);
    if (to)
      for (int k = 0; k < 3; ++k) { to->top[k] += fp.top[k]; to->bot[k] += fp.bot[k]; }
  }
  if (M.floating) { /* the base's own I_b a_b + v_b x* (I_b v_b), base frame */
    Sv Ia, Iv, bias;
    abi_mul(&st->base_abi, &ab, &Ia);
    abi_mul(&st->base_abi, &st->base_velocity, &Iv);
    sv_cross_force(&st->base_velocity, &Iv, &bias);
    for (int k = 0; k < 3; ++k) {
      tau[k] = fb.top[k] + Ia.top[k] + bias.top[k];
      tau[3 + k] = fb.bot[k] + Ia.bot[k] + bias.bot[k];
    }
  }
  return 0;
}
