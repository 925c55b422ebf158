/* TEST INFRASTRUCTURE - NOT PRODUCT CODE, never loaded by the package.
 *
 * Link velocities and accelerations IN LINK FRAMES on the C oracle: oracle/tds_oracle.c is included as it stands, its static
 * forward_kinematics(q, qd) gives every link's X_world, X_parent, S, v and c = v x vJ; then the accelerations root to leaf,
 * a_i = X_i a_parent + S_i qdd_i + c_i (kinematics.hpp:18-148 with qdd), from the base's a = qdd[0:6] (floating) or 0, without gravity.
 * Independent of the kernel's common-frame arithmetic.  Bound by tests/emu_point_motion.py.
 *   gcc -std=c11 -O2 -fPIC -shared -I<include> -I<oracle> tests/cpp/oracle_motion.c -o tests/cpp/_oracle_motion.so -lm */
#include "../../oracle/tds_oracle.c"

/* out [n_links + 1][24], record 0 the base and record i + 1 link i: the world rotation R [9] (row-major, link to world), the origin in
 * world coordinates [3], the spatial velocity v [6] and acceleration a [6] ([angular; linear at the origin], link axes) at q, qd, qdd
 * (qd, qdd NULL: zero).  Returns 0, or < 0. */
int tdso_motion(const double* model, const double* q, const double* qd, const double* qdd, double* out) {
  static Sv a[MAXL];
  Model M;
  int rc = model_open(model, &M);
  if (rc) return rc;
  State* st = &g_state;
  forward_kinematics(&M, st, q, qd);
  Sv ab, vb;
  for (int k = 0; k < 3; ++k) {
    ab.top[k] = (M.floating && qdd) ? qdd[k] : 0.0;
    ab.bot[k] = (M.floating && qdd) ? qdd[3 + k] : 0.0;
  }
  if (M.floating) vb = st->base_velocity;
  else memset(&vb, 0, sizeof vb);
  for (int i = 0; i < M.n_links; ++i) {
    const double* l = LNK(&M, i);
    const int parent = (int)l[TDSM_L_PARENT];
    Sv xa;
    xf_apply_motion(&st->X_parent[i], parent >= 0 ? &a[parent] : &ab, &xa);
    const double qddv = ((int)l[TDSM_L_JTYPE] == TDSJ_FIXED || !qdd) ? 0.0 : qdd[(int)l[TDSM_L_QDIDX]];
    for (int k = 0; k < 3; ++k) {
      a[i].top[k] = xa.top[k] + st->c[i].top[k] + st->S[i].top[k] * qddv;
      a[i].bot[k] = xa.bot[k] + st->c[i].bot[k] + st->S[i].bot[k] * qddv;
    }
  }
  for (int b = 0; b <= M.n_links; ++b) {
    const Xf* X = b == 0 ? &st->base_X_world : &st->X_world[b - 1];
    const Sv* v = b == 0 ? &vb : &st->v[b - 1];
    const Sv* ac = b == 0 ? &ab : &a[b - 1];
    double* o = out + (size_t)b * 24;
    memcpy(o, X->R, 9 * sizeof(double));
    memcpy(o + 9, X->t, 3 * sizeof(double));
    memcpy(o + 12, v->top, 3 * sizeof(double));
    memcpy(o + 15, v->bot, 3 * sizeof(double));
    memcpy(o + 18, ac->top, 3 * sizeof(double));
    memcpy(o + 21, ac->bot, 3 * sizeof(double));
  }
  return 0;
}
