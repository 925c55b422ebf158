/* TEST INFRASTRUCTURE - NOT PRODUCT CODE, never loaded by the package.
 *
 * The C oracle's point Jacobian: oracle/tds_oracle.c is included as it stands, and its static forward_kinematics and point_jacobian
 * (jacobian.hpp:13-83) are exported as tdso_point_jacobian.  Link transforms at q come from the oracle's own tdso_step (MODE_FD with
 * zero qd, link_xf_out), which this library exports too.  Bound by tests/emu_kin.py.
 *   gcc -std=c11 -O2 -fPIC -shared -I<include> -I<oracle> tests/cpp/oracle_kin.c -o tests/cpp/_oracle_kin.so -lm */
#include "../../oracle/tds_oracle.c"

/* J [3][n_qd] (row-major) of the world point `point_world` on link `link` (-1: the base) at q: forward_kinematics(q, NULL), then
 * point_jacobian.  Returns 0, or < 0. */
int tdso_point_jacobian(const double* model, const double* q, int link, const double* point_world, double* J) {
  Model M;
  int rc = model_open(model, &M);
  if (rc) return rc;
  if (link < -1 || link >= M.n_links) return -10;
  forward_kinematics(&M, &g_state, q, 0);
  point_jacobian(&M, &g_state, link, point_world, J);
  return 0;
}
