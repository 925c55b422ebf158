/* C-ABI of libtds_b200.so: the batched rigid-body env-step for the H100.
 *
 * Plain pointers and sizes only (no torch / C++ types).  Each entry point cites the reference
 * interface it replaces (paths relative to erwincoumans/tiny-differentiable-simulator @ 8381b8c).
 * INTEGRATION.md shows the reference-side bindings (dlopen of the v1 symbols, a
 * CustomForwardDynamicsStepper subclass, a pybind shim).
 *
 * Device-side state is SoA fp32: array[dim][n_stride], environment index fastest
 * (n_stride = n_envs rounded up to 32), so a warp of 32 environments reads 128 contiguous bytes
 * per coordinate.
 */
#ifndef TDS_B200_H
#define TDS_B200_H
#ifndef __cplusplus
#include <stdbool.h>
#endif
#ifdef __cplusplus
extern "C" {
#endif

typedef struct tds_b200_sim tds_b200_sim;

/* pipeline selector of tds_b200_step_* */
#define TDS_B200_MODE_FD 0        /* tds::forward_dynamics only, src/dynamics/forward_dynamics.hpp:11 (qdd out) */
#define TDS_B200_MODE_NOCONTACT 1 /* FD -> integrate_euler, examples/environments/cartpole_environment2.h:86-93 */
#define TDS_B200_MODE_FULL 2      /* FD -> integrate_euler_qdd -> World::step -> integrate_euler,
                                     examples/environments/locomotion_contact_simulation.h:261-269 */

#define TDS_B200_MODE_WORLD 3     /* World::step(dt) alone, src/world.hpp:302-363: contact detection + constraint solve on the
                                     given (q, qd); qd out, q unchanged.  Stage of the fine-grained pytinydiffsim sequence
                                     forward_dynamics -> integrate_euler_qdd -> world.step -> integrate_euler
                                     (python/pytinydiffsim.inl:659-663,857-876) */

/* arithmetic selector */
#define TDS_B200_PREC_MIXED 0 /* default: fp32 ABA / factorisation / PGS; fp64 kinematics, contact geometry,
                                 composite inertias, CRBA products, Jacobians and LCP right-hand side */
#define TDS_B200_PREC_F64 1   /* strict: every stage fp64; meets 1e-5 on every model of the parity suite */
#define TDS_B200_PREC_F32 2   /* comparison only (the reference's own fp32 build misses the tolerance) */
#define TDS_B200_PREC_AUTO (-1) /* default: MIXED for a model the library holds a compiled, parity-validated instance of
                                   (Laikago, Ant), F64 otherwise */

const char* tds_b200_last_error(void);

/* ---- model compiler (setup time) -------------------------------------------------------------
 * Replaces UrdfCache::construct -> UrdfParser::load_urdf + UrdfToMultiBody::convert_to_multi_body
 * (src/urdf/urdf_cache.hpp:74-84, src/urdf/urdf_parser.hpp:707-925, src/urdf/urdf_to_multi_body.hpp:41).
 * urdf / plane_urdf: file path or URDF text (text if the first non-blank char is '<'); plane_urdf may
 * be NULL/"" for a world without ground plane.  Writes the flat model (include/tds_b200_model.h);
 * returns its length in doubles (call with out=NULL to size), <0 on error. */
int tds_b200_urdf_to_model(const char* urdf, const char* plane_urdf, int floating, double* out, int cap);

/* ---- simulator lifecycle ----------------------------------------------------------------------
 * One sim = n_envs independent copies of World{plane, MultiBody} (src/world.hpp:41, multi_body.hpp:13)
 * resident on CUDA device `device`.  Returns NULL on error (see tds_b200_last_error). */
tds_b200_sim* tds_b200_create(const double* model, int n_model_doubles, int n_envs, int device);
/* Host-only acceptance check of a flat model (no GPU needed): 0, or the negative code tds_b200_create would fail with
 * (mesh shapes against the plane, spherical joints with a stiffness, capacity); the reason is in tds_b200_last_error(). */
int tds_b200_validate_model(const double* model, int n_model);
void tds_b200_destroy(tds_b200_sim* sim);

/* World / solver parameters: World::{default_friction,default_restitution} (src/world.hpp:68-69),
 * gravity (world.hpp:50), MultiBodyConstraintSolver::{erp_,cfm_,pgs_iterations_,keep_all_points_}
 * (src/mb_constraint_solver.hpp:59-70).  Defaults equal the reference's. */
int tds_b200_set_params(tds_b200_sim* sim, double dt, const double gravity[3], double friction, double restitution,
                        double erp, double cfm, int pgs_iterations, int keep_all_points);

/* Contact law.  0 (default): the reference's impulse-level LCP solved by projected Gauss-Seidel
 * (MultiBodyConstraintSolver, src/mb_constraint_solver.hpp).  1: spring-damper contacts - the reference's
 * MultiBodyConstraintSolverSpring, whose SOURCE IS ABSENT from the snapshot (only the parameter names survive,
 * python/pytinydiffsim.inl:825-856: spring_k, damper_d, exponent_n, hard_contact_condition, v_transition, ...), so the law
 * is the one written down in DESIGN.md "Spring-damper contacts" (Hunt-Crossley normal force k x^n + d x^n xdot, clamped at
 * 0 with hard_contact_condition; friction mu f_n tanh(|v_t| / v_transition) against the tangential velocity; applied as
 * impulses f dt through M^-1 Jc^T): PARITY UNPINNED, self-consistent with oracle/tds_oracle.c. */
int tds_b200_set_contact_model(tds_b200_sim* sim, int contact_model, double spring_k, double damper_d, double exponent_n,
                               double v_transition, int hard_contact_condition);

/* PD / environment parameters of LocomotionContactSimulation
 * (examples/environments/locomotion_contact_simulation.h:28-48,168-258): action k drives the k-th
 * non-fixed link at or after `start_link` (base_dof_) towards initial_poses[k] + clamp(action, +-limit).
 * reward_kind: 0 none, 1 Laikago fixed-base emulation, 2 floating, 3 Ant fixed-base emulation (ant_environment2.h:75-105)
 * (examples/environments/laikago_environment2.h:130-171). */
int tds_b200_set_env(tds_b200_sim* sim, int n_act, const double* initial_poses, int start_link, double kp,
                     double kd, double max_force, double action_limit, int reward_kind);

/* VectorizedEnvironment's auto_reset_when_done (examples/ars/ars_vectorized_environment.h:262-283) on the
 * device: an environment that reports done is put back to reset_q[n_q] with zero velocity at the end of
 * that step (the reward/done outputs of the step are kept).  The host-side reset() of the Python mirror adds
 * the reference's joint noise and settle steps (laikago_environment2.h:63-116). */
int tds_b200_set_auto_reset(tds_b200_sim* sim, int enable, const double* reset_q);

int tds_b200_set_precision(tds_b200_sim* sim, int precision);
int tds_b200_get_precision(const tds_b200_sim* sim);   /* the resolved selector (never AUTO) */
/* Name of the step kernel the last tds_b200_step_* call launched (selection: DESIGN.md "Kernel selection"). */
const char* tds_b200_kernel_name(const tds_b200_sim* sim);

/* dims[0..7] = n_envs, n_stride, n_q (MultiBody::dof), n_qd (dof_qd), n_tau (dof_actuated), n_links,
 *              n_contact_points, n_act */
int tds_b200_get_dims(const tds_b200_sim* sim, int dims[8]);

/* ---- device-resident fast path -------------------------------------------------------------------
 * One launch = one step of all environments.  Pointers are DEVICE pointers to SoA fp32 arrays
 * [dim][n_stride]; q_in/qd_in may alias q_out/qd_out.  `tau_or_action`: [n_tau][n_stride] joint torques
 * (MultiBody::tau_, multi_body.hpp:86) when use_pd == 0, else [n_act][n_stride] policy actions.
 * Optional outputs may be NULL: qdd_out [n_qd][ns] (MODE_FD), reward/done [n_stride],
 * contact_dist [n_contact_points][ns] (ContactPoint::distance of every candidate point in the
 * reference's enumeration order, src/world.hpp:212-281), link_xf [n_links*12][ns].
 * stream: a cudaStream_t (NULL = default stream).  Asynchronous.  Returns a cudaError_t value. */
int tds_b200_step_device(tds_b200_sim* sim, int mode, int use_pd, const float* q_in, const float* qd_in,
                         const float* tau_or_action, float* q_out, float* qd_out, float* qdd_out, float* reward,
                         float* done, float* contact_dist, float* link_xf, void* stream);

/* ---- differentiable step (SURVEY 8f.4; the role of <model>_jacobian in the reference's generated libraries,
 * src/utils/cuda/cuda_codegen.hpp:303-426, there produced by CppAD from the recorded tape) -----------------------------
 * Dense Jacobian of one step per environment by forward-mode dual numbers (fp64) through the step kernel: rows = q' | qd'
 * (modes NOCONTACT / FULL) or qdd (mode FD); columns = q | qd | tau (use_pd == 0) or q | qd | action | kp, kd, max_force
 * (use_pd == 1: the input vector of LocomotionContactSimulation, locomotion_contact_simulation.h:160-166).  Derivatives
 * are those of the branch taken (contact set, clamps).  dims[0..1] = rows, columns.
 *   device: q, qd, tau_or_action as in tds_b200_step_device; jac [rows * cols][n_stride] fp64 (row-major per environment)
 *   host:   q [n][n_q], qd [n][n_qd], tau_or_action [n][..] fp64; jac [n][rows][cols] fp64 */
int tds_b200_jacobian_dims(const tds_b200_sim* sim, int mode, int use_pd, int dims[2]);
int tds_b200_step_jacobian_device(tds_b200_sim* sim, int mode, int use_pd, const float* q, const float* qd,
                                  const float* tau_or_action, double* jac, void* stream);
int tds_b200_step_jacobian_host(tds_b200_sim* sim, int mode, int use_pd, const double* q, const double* qd,
                                const double* tau_or_action, double* jac);

/* Vector-Jacobian product of one step per environment, g_in = g_out^T J with J, rows and columns as above, by reverse mode:
 * the step kernel on a taping fp64 scalar, one lane per environment, then a reverse sweep in the same lane (DESIGN.md 7.8).
 * The gradient is that of the fp64 world-frame step at the fp32-rounded inputs, of the branch taken.  Argument checks as for
 * the Jacobian: mode WORLD -> -2, use_pd without tds_b200_set_env -> -3, a NULL required pointer -> -1.
 *   device: q, qd, tau_or_action as in tds_b200_step_device; g_out [rows][n_stride], g_in [cols][n_stride] fp64.  Environments
 *           run in chunks of at most 2 GB of tape; the call synchronises its stream after every chunk (it reads the tape's
 *           overflow flag, and reruns a chunk with twice the capacity when it is set; the capacity stays grown).
 *   host:   q [n][n_q], qd [n][n_qd], tau_or_action [n][n_tau | n_act] fp64 (rounded to fp32 before the step),
 *           g_out [n][rows], g_in [n][cols] fp64.  Synchronous.
 * tds_b200_vjp_tape_info: info[0] = tape capacity in use (nodes per lane), info[1] = environments per chunk at that capacity
 * (a batch of more environments runs in several chunks). */
int tds_b200_step_vjp_device(tds_b200_sim* sim, int mode, int use_pd, const float* q, const float* qd, const float* tau_or_action,
                             const double* g_out, double* g_in, void* stream);
int tds_b200_step_vjp_host(tds_b200_sim* sim, int mode, int use_pd, const double* q, const double* qd,
                           const double* tau_or_action, const double* g_out, double* g_in);
int tds_b200_vjp_tape_info(const tds_b200_sim* sim, int info[2]);

/* ---- per-environment physical parameters (DESIGN.md 7.9): system identification and domain randomisation ----------------------
 * Parameter ids over the flat model (for a world of several multibodies: the links of the merged model):
 *   0                              friction (World::default_friction; SimParams friction)
 *   1                              restitution (World::default_restitution)
 *   2 + 10 b + c                   body b: b = 0 the floating base (floating models only), b = i + 1 link i;
 *                                  c = mass, com x, com y, com z, inertia about the com xx, xy, xz, yy, yz, zz (off-diagonal ids are
 *                                  the symmetric component: the value stands for both entries)
 *   2 + 10 (n_links + 1) + 2 i + c link i: c = 0 joint stiffness, c = 1 joint damping (used at fp32, as the model stores them)
 * tds_b200_param_count: the number of ids, 2 + 10 (n_links + 1) + 2 n_links.
 *
 * tds_b200_set_physical_params_*: install k parameters; the simulator copies the values into a buffer it owns.  device: values
 * [k][n_stride] fp64 device pointer, copied on `stream`; host: values [n][k] fp64, synchronous.  k = 0 clears the set.  Refused (-2,
 * reason in tds_b200_last_error): an id out of range, an id given twice, a base id on a fixed-base model.  While a set is installed
 * every stepping entry point (step, Jacobian, VJP, env_step_*, env_reset settle steps, rollouts, ars_train_step, the visual stream)
 * uses each environment's values for those ids and the model's values for the rest, on the generic world-frame kernel.  Installing
 * another set of ids, clearing it or growing its buffer drops the captured graphs of tds_b200_env_step_host; new values for the
 * same ids keep the buffer, so a captured graph sees them.
 *
 * tds_b200_step_param_jacobian_*: d(outputs) / d(installed parameters) by dual numbers, rows as tds_b200_step_jacobian_*, k columns
 * (k directions per environment).  device: jac [rows * k][n_stride]; host: jac [n][rows][k].  -4 when no set is installed.
 * tds_b200_step_vjp_params_*: the reverse sweep of tds_b200_step_vjp_*, which also writes g_par = g_out^T d(outputs) / d(parameters):
 * device [k][n_stride], host [n][k].  g_in may be NULL.  Argument checks as for the VJP; -4 when no set is installed. */
int tds_b200_param_count(const tds_b200_sim* sim);
int tds_b200_set_physical_params_device(tds_b200_sim* sim, int k, const int* ids, const double* values, void* stream);
int tds_b200_set_physical_params_host(tds_b200_sim* sim, int k, const int* ids, const double* values);
int tds_b200_step_param_jacobian_device(tds_b200_sim* sim, int mode, int use_pd, const float* q, const float* qd,
                                        const float* tau_or_action, double* jac, void* stream);
int tds_b200_step_param_jacobian_host(tds_b200_sim* sim, int mode, int use_pd, const double* q, const double* qd,
                                      const double* tau_or_action, double* jac);
int tds_b200_step_vjp_params_device(tds_b200_sim* sim, int mode, int use_pd, const float* q, const float* qd,
                                    const float* tau_or_action, const double* g_out, double* g_in, double* g_par, void* stream);
int tds_b200_step_vjp_params_host(tds_b200_sim* sim, int mode, int use_pd, const double* q, const double* qd,
                                  const double* tau_or_action, const double* g_out, double* g_in, double* g_par);

/* ---- Jacobian-vector products (forward mode, DESIGN.md 7.10): t_out = J V for m tangent directions V per environment ----------
 * J is the step's Jacobian over its inputs (columns as tds_b200_step_jacobian_*, kp, kd, max_force included with use_pd) and, while a
 * parameter set is installed, over the installed parameters (in the order of tds_b200_set_physical_params_*).  Semantics as the
 * Jacobian's: the derivative of the fp64 world-frame step at the fp32-rounded inputs, of the branch taken, with each environment's
 * parameter values.  One lane per (environment, tangent) of the dual-number step; the tangents run in chunks as the Jacobian's
 * directions, so m = cols costs about one Jacobian.  t_in or t_par may be NULL (zero tangent), not both.  Argument checks: mode WORLD
 * -> -2, use_pd without tds_b200_set_env -> -3, a NULL required pointer (q, qd, t_out; the action with use_pd), m < 1 or both tangents
 * NULL -> -1, t_par without an installed set -> -4.
 *   device: q, qd, tau_or_action as in tds_b200_step_device; t_in [cols * m][n_stride], t_par [k * m][n_stride], t_out [rows * m][n_stride]
 *           fp64: entry (c, j) of environment e at (c * m + j) * n_stride + e.  Asynchronous on `stream`.
 *   host:   q [n][n_q], qd [n][n_qd], tau_or_action [n][..] fp64 (rounded to fp32); t_in [n][cols][m], t_par [n][k][m],
 *           t_out [n][rows][m] fp64.  Synchronous.
 * tds_b200_jacobian_chunk: the directions (Jacobian columns or tangents) one launch takes; more run in several launches, each with
 * arena scratch of at most 2 GB. */
int tds_b200_step_jvp_device(tds_b200_sim* sim, int mode, int use_pd, const float* q, const float* qd, const float* tau_or_action,
                             int m, const double* t_in, const double* t_par, double* t_out, void* stream);
int tds_b200_step_jvp_host(tds_b200_sim* sim, int mode, int use_pd, const double* q, const double* qd, const double* tau_or_action,
                           int m, const double* t_in, const double* t_par, double* t_out);
int tds_b200_jacobian_chunk(const tds_b200_sim* sim);

/* ---- joint-space mass matrix M(q) (DESIGN.md 7.12; mass_matrix in python/pytinydiffsim.inl) ----------------------------------------
 * The dense symmetric n_qd x n_qd matrix of every environment, both triangles, by the CRBA of the world-frame step (the matrix its
 * contact solve factors), in fp64 at the fp32-rounded q; qd plays no part (the reference calls forward_kinematics with an empty qd).
 * A world of several multibodies gives the block-diagonal matrix.  While a parameter set is installed, each environment's masses,
 * centres of mass and inertias are used; stiffness, damping, friction and restitution do not enter M (their derivative is zero).
 * Argument checks: a NULL required pointer, m < 1 or both tangents NULL -> -1; t_par / g_par without an installed set -> -4.
 *   device: q [n_q][n_stride] fp32 as tds_b200_step_device; M [n_qd * n_qd][n_stride] fp64, entry (r, c) at (r * n_qd + c) * n_stride + e.
 *           Asynchronous on `stream`.
 *   host:   q [n][n_q] fp64 (rounded to fp32); M [n][n_qd][n_qd] fp64.  Synchronous.
 * _jvp: dM = sum_c dM/dq_c t_q[c] + sum_s dM/dp_s t_par[s] for m tangents, one lane per (environment, tangent) of the dual-number
 *   instance, in chunks as tds_b200_step_jvp_*.  M (may be NULL) receives the value.  Layouts as tds_b200_step_jvp_*: device t_q
 *   [n_q * m][n_stride], t_par [k * m][n_stride], t_M [n_qd * n_qd * m][n_stride] (entry ((r n_qd + c), j) at ((r n_qd + c) m + j) n_stride + e);
 *   host t_q [n][n_q][m], t_par [n][k][m], t_M [n][n_qd][n_qd][m].
 * _vjp: g_q[c] = sum_rs G[r][s] dM[r][s]/dq_c and, while a set is installed, g_par[s] = sum G dM/dp_s, for a cotangent G in M's
 *   layout: the JVP along the n_q + k identity tangents contracted with G on the device.  g_q or g_par may be NULL, not both.  Device
 *   g_q [n_q][n_stride], g_par [k][n_stride] fp64 (asynchronous); host g_q [n][n_q], g_par [n][k] (synchronous). */
int tds_b200_mass_matrix_device(tds_b200_sim* sim, const float* q, double* M, void* stream);
int tds_b200_mass_matrix_host(tds_b200_sim* sim, const double* q, double* M);
int tds_b200_mass_matrix_jvp_device(tds_b200_sim* sim, const float* q, int m, const double* t_q, const double* t_par, double* M,
                                    double* t_M, void* stream);
int tds_b200_mass_matrix_jvp_host(tds_b200_sim* sim, const double* q, int m, const double* t_q, const double* t_par, double* M,
                                  double* t_M);
int tds_b200_mass_matrix_vjp_device(tds_b200_sim* sim, const float* q, const double* G, double* g_q, double* g_par, void* stream);
int tds_b200_mass_matrix_vjp_host(tds_b200_sim* sim, const double* q, const double* G, double* g_q, double* g_par);

/* ---- forward kinematics and linear point Jacobians (DESIGN.md 7.13; forward_kinematics_q, point_jacobian: jacobian.hpp:13-83) ------
 * From q alone (rounded to fp32; qd plays no part) and a point table of K points (0 <= K <= TDS_B200_MAX_KIN_POINTS), the same for all
 * environments and passed with each call in host memory: point k sits on link links[k] (-1: the base) at local[3k .. 3k+2] in that
 * link's frame.  Outputs, fp64, world coordinates, each may be NULL but not all three:
 *   xf: every link's world transform, 12 per link (R row-major, then the position: the layout of tds_b200_step's link transforms);
 *   x:  every point's world position;
 *   J:  every point's 3 x n_qd linear Jacobian, the reference's convention: a floating base gives the columns [-[x - r0]x^T | I3]
 *       with the base's rotation ignored; fixed links have no columns; a spherical joint has 3; in a world of several multibodies a
 *       point has entries in its own multibody's dofs only.
 * Installed physical parameters do not enter kinematics.  Argument checks -> -1: NULL q; K out of range, a link index out of range,
 * or NULL links / local with K > 0; no output (no cotangent); m < 1 or NULL t_q; NULL g_q.
 *   device: q [n_q][n_stride] fp32 as tds_b200_step_device; xf [n_links * 12][n_stride], x [3K][n_stride], J [3K * n_qd][n_stride] fp64
 *           with entry (point k, row r, column c) of J at row (3k + r) * n_qd + c.  Asynchronous on `stream`.
 *   host:   q [n][n_q] fp64; xf [n][n_links][12], x [n][K][3], J [n][K][3][n_qd].  Synchronous.
 * _jvp: the directional derivatives along m tangents t_q of q, one lane per (environment, tangent) of the dual-number instance, in
 *   chunks as tds_b200_step_jvp_*.  Device t_q [n_q * m][n_stride] and t_xf / t_x / t_J [rows * m][n_stride] (entry (r, j) at
 *   (r * m + j) * n_stride + e); host t_q [n][n_q][m], t_xf [n][n_links * 12][m], t_x [n][3K][m], t_J [n][3K * n_qd][m].
 * _vjp: g_q[c] = <G_xf, dxf/dq_c> + <G_x, dx/dq_c> + <G_J, dJ/dq_c> for cotangents in the outputs' layouts (a NULL one is zero): the
 *   JVP along the n_q identity tangents contracted with the cotangent on the device.  Device g_q [n_q][n_stride] fp64 (asynchronous);
 *   host g_q [n][n_q] (synchronous). */
#define TDS_B200_MAX_KIN_POINTS 64
int tds_b200_kinematics_device(tds_b200_sim* sim, const float* q, int K, const int* links, const double* local, double* xf, double* x,
                               double* J, void* stream);
int tds_b200_kinematics_host(tds_b200_sim* sim, const double* q, int K, const int* links, const double* local, double* xf, double* x,
                             double* J);
int tds_b200_kinematics_jvp_device(tds_b200_sim* sim, const float* q, int K, const int* links, const double* local, int m,
                                   const double* t_q, double* t_xf, double* t_x, double* t_J, void* stream);
int tds_b200_kinematics_jvp_host(tds_b200_sim* sim, const double* q, int K, const int* links, const double* local, int m,
                                 const double* t_q, double* t_xf, double* t_x, double* t_J);
int tds_b200_kinematics_vjp_device(tds_b200_sim* sim, const float* q, int K, const int* links, const double* local, const double* G_xf,
                                   const double* G_x, const double* G_J, double* g_q, void* stream);
int tds_b200_kinematics_vjp_host(tds_b200_sim* sim, const double* q, int K, const int* links, const double* local, const double* G_xf,
                                 const double* G_x, const double* G_J, double* g_q);

/* ---- inverse dynamics tau = ID(q, qd, qdd) and bias forces (DESIGN.md 7.14; inverse_dynamics.hpp) ------------------------------------
 * The joint forces tau [n_qd] (fp64, one row per dof, a floating base's 6 rows included) for which the multibody has the accelerations
 * qdd, by the recursive Newton-Euler algorithm at the fp32-rounded q, qd, qdd and the simulator's gravity (tds_b200_set_params).  qd or
 * qdd may be NULL, meaning zero; bias forces h(q, qd) are ID(q, qd, 0): pass a NULL qdd.
 *   Fixed base (worlds of several multibodies included): the exact inverse of this library's forward dynamics (MODE_FD), so tau
 *   contains the terms the ABA subtracts: stiffness q + damping qd of 1-dof joints, the quaternion axis-angle stiffness term and per-dof
 *   damping of spherical joints.  While a parameter set is installed, each environment's masses, centres of mass, inertias, stiffness
 *   and damping are used.
 *   Floating base: the textbook RNEA in the coordinates of tds_b200_mass_matrix: qdd[0:6] is the base-frame spatial acceleration
 *   [angular; linear], gravity is rotated into the base frame, and rows 0..5 are the wrench on the base in the base frame [moment
 *   about the base origin; force].  This is NOT the inverse of the reference's floating-base forward dynamics, which adds gravity
 *   un-rotated, has a frame-mixing gyroscopic term and does not invert its own mass matrix.
 * Argument checks: NULL q, no output (tau, t_tau; G, or every cotangent output), m < 1 or every tangent NULL -> -1; t_par / g_par
 * without an installed set -> -4.
 *   device: q [n_q][n_stride], qd and qdd [n_qd][n_stride] fp32 as tds_b200_step_device; tau [n_qd][n_stride] fp64.  Asynchronous.
 *   host:   q [n][n_q], qd and qdd [n][n_qd] fp64 (rounded to fp32); tau [n][n_qd] fp64.  Synchronous.
 * _jvp: dtau along m tangents of q, qd, qdd and the installed parameters (each may be NULL: zero, not all), one lane per (environment,
 *   tangent) of the dual-number instance, in chunks as tds_b200_step_jvp_*.  tau (may be NULL) receives the value.  Device t_q
 *   [n_q * m][n_stride], t_qd and t_qdd [n_qd * m][n_stride], t_par [k * m][n_stride], t_tau [n_qd * m][n_stride] (entry (r, j) at
 *   (r * m + j) * n_stride + e); host t_q [n][n_q][m], t_qd and t_qdd [n][n_qd][m], t_par [n][k][m], t_tau [n][n_qd][m].
 * _vjp: g_x[c] = sum_r G[r] dtau[r]/dx_c for x = q, qd, qdd and, while a set is installed, the parameters, for a cotangent G in tau's
 *   layout: the JVP along the n_q + 2 n_qd (+ k) identity tangents contracted with G on the device.  Any of g_q, g_qd, g_qdd, g_par may
 *   be NULL, not all.  Device g_q [n_q][n_stride], g_qd and g_qdd [n_qd][n_stride], g_par [k][n_stride] fp64 (asynchronous); host
 *   g_q [n][n_q], g_qd and g_qdd [n][n_qd], g_par [n][k] (synchronous). */
int tds_b200_inverse_dynamics_device(tds_b200_sim* sim, const float* q, const float* qd, const float* qdd, double* tau, void* stream);
int tds_b200_inverse_dynamics_host(tds_b200_sim* sim, const double* q, const double* qd, const double* qdd, double* tau);
int tds_b200_inverse_dynamics_jvp_device(tds_b200_sim* sim, const float* q, const float* qd, const float* qdd, int m, const double* t_q,
                                         const double* t_qd, const double* t_qdd, const double* t_par, double* tau, double* t_tau,
                                         void* stream);
int tds_b200_inverse_dynamics_jvp_host(tds_b200_sim* sim, const double* q, const double* qd, const double* qdd, int m, const double* t_q,
                                       const double* t_qd, const double* t_qdd, const double* t_par, double* tau, double* t_tau);
int tds_b200_inverse_dynamics_vjp_device(tds_b200_sim* sim, const float* q, const float* qd, const float* qdd, const double* G, double* g_q,
                                         double* g_qd, double* g_qdd, double* g_par, void* stream);
int tds_b200_inverse_dynamics_vjp_host(tds_b200_sim* sim, const double* q, const double* qd, const double* qdd, const double* G, double* g_q,
                                       double* g_qd, double* g_qdd, double* g_par);

/* ---- centre of mass, centroidal momentum matrix and its bias (DESIGN.md section 7.16) -------------------------------------------------
 * At the fp32-rounded q and qd (qd may be NULL, meaning zero), fp64 outputs, each of which may be NULL (not all three):
 *   com [10]: the body record of the whole system in the order of the parameter ids' body record: the total mass m, the centre of mass
 *     c [3] in world coordinates, the rotational inertia I_G about c in world axes [6] (xx, xy, xz, yy, yz, zz).  The counted bodies are
 *     the links and a floating base; a fixed base belongs to the world and is not counted.
 *   A [6 n_qd]: the centroidal momentum matrix A_G, entry (r, c) at r * n_qd + c.  Rows: [angular momentum about c; linear momentum] in
 *     world axes; columns: the coordinates of tds_b200_mass_matrix (a floating base's qd[0:6] is the base-frame twist [w; v]).  So the
 *     centroidal momentum is h_G = A qd and the Jacobian of c is A[3:6] / m.
 *   bias [6]: A_G' qd, the rate of h_G when qdd = 0, rows and axes as A.  Velocity terms only: gravity, joint stiffness and damping do
 *     not enter.  With every external wrench W about c, A qdd + bias = sum W + [0; m g].
 * While a parameter set is installed, each environment's masses, centres of mass and inertias (links and floating base) are used;
 * friction, restitution, stiffness and damping do not enter.  An environment whose installed masses do not sum to a positive value
 * gets non-finite c and I_G.
 * Argument checks: NULL q, no output, m < 1, every tangent NULL, no cotangent or no cotangent output -> -1; a world of several
 * multibodies (TDSM_H_NBODIES > 1) or a model whose counted bodies have zero total mass -> -2; t_par / g_par without an installed set
 * -> -4.
 *   device: q [n_q][n_stride], qd [n_qd][n_stride] fp32; com [10][n_stride], A [6 n_qd][n_stride], bias [6][n_stride].  Asynchronous.
 *   host:   q [n][n_q], qd [n][n_qd] fp64 (rounded to fp32); com [n][10], A [n][6 n_qd], bias [n][6].  Synchronous.
 * _jvp: the outputs' derivatives along m tangents of q, qd and the installed parameters (each may be NULL: zero, not all), as
 *   tds_b200_inverse_dynamics_jvp_*.  Device t_q [n_q * m][n_stride], t_qd [n_qd * m][n_stride], t_par [k * m][n_stride], t_com
 *   [10 m][n_stride], t_A [6 n_qd m][n_stride], t_bias [6 m][n_stride] (entry (r, j) at (r * m + j) * n_stride + e); host t_q
 *   [n][n_q][m], t_qd [n][n_qd][m], t_par [n][k][m], t_com [n][10][m], t_A [n][6 n_qd][m], t_bias [n][6][m].  NULL outputs are skipped.
 * _vjp: g_x[c] = <G, d(com | A | bias)/dx_c> for x = q, qd and, while a set is installed, the parameters, for cotangents G_com, G_A,
 *   G_bias in the outputs' layouts (NULL: zero, not all): the JVP along the n_q + n_qd (+ k) identity tangents contracted with G on the
 *   device.  Any of g_q, g_qd, g_par may be NULL, not all.  Device g_q [n_q][n_stride], g_qd [n_qd][n_stride], g_par [k][n_stride] fp64
 *   (asynchronous); host g_q [n][n_q], g_qd [n][n_qd], g_par [n][k] (synchronous). */
int tds_b200_centroidal_device(tds_b200_sim* sim, const float* q, const float* qd, double* com, double* A, double* bias, void* stream);
int tds_b200_centroidal_host(tds_b200_sim* sim, const double* q, const double* qd, double* com, double* A, double* bias);
int tds_b200_centroidal_jvp_device(tds_b200_sim* sim, const float* q, const float* qd, int m, const double* t_q, const double* t_qd,
                                   const double* t_par, double* t_com, double* t_A, double* t_bias, void* stream);
int tds_b200_centroidal_jvp_host(tds_b200_sim* sim, const double* q, const double* qd, int m, const double* t_q, const double* t_qd,
                                 const double* t_par, double* t_com, double* t_A, double* t_bias);
int tds_b200_centroidal_vjp_device(tds_b200_sim* sim, const float* q, const float* qd, const double* G_com, const double* G_A,
                                   const double* G_bias, double* g_q, double* g_qd, double* g_par, void* stream);
int tds_b200_centroidal_vjp_host(tds_b200_sim* sim, const double* q, const double* qd, const double* G_com, const double* G_A,
                                 const double* G_bias, double* g_q, double* g_qd, double* g_par);

/* ---- spatial point Jacobians, point velocities and accelerations J qdd + J' qd (DESIGN.md section 7.17; kinematics.hpp:18-148) ------
 * At the fp32-rounded q, qd and qdd (qd or qdd may be NULL, meaning zero), for the point table of tds_b200_kinematics_* (K points,
 * 0 <= K <= TDS_B200_MAX_KIN_POINTS, point k on links[k] (-1: the base) at local[3k .. 3k+2] in that link's frame, host memory), fp64
 * outputs in world axes, each may be NULL but not all three:
 *   J [6 n_qd] per point: the spatial point Jacobian, rows [w; x'] with [w; x'] = J qd, entry (point k, row r, column c) at row
 *     (6k + r) * n_qd + c.  A joint column is [S.top; S.bot + S.top x (x - O)] for the joint's world motion subspace S at the world
 *     origin O, so the linear rows equal tds_b200_kinematics' J on the joint columns.  Fixed links have no columns, a spherical joint has
 *     3; in a world of several multibodies a point has entries in its own multibody's dofs only.
 *     FLOATING BASE - unlike tds_b200_kinematics: the columns are the coordinates of tds_b200_mass_matrix, inverse_dynamics and
 *     centroidal, where qd[0:6] is the base-frame twist [w_b; v_b] and qdd[0:6] its time derivative.  The base columns are [R_b | 0] in
 *     the angular rows and [-[x - p_b]x R_b | R_b] in the linear rows (p_b the base position), i.e. tds_b200_kinematics' base columns
 *     times diag(R_b, R_b), whose reference convention ignores the base rotation.  With these columns J composes with M, h and A.
 *   vel [6] per point: [w; x'], the angular velocity of the point's link and the velocity of the point's world position x.
 *   acc [6] per point: [w'; x''], the time derivatives of w and of x (classical, not spatial, acceleration): acc = J qdd + J' qd, and
 *     with qdd = NULL the drift J' qd.
 * Gravity does not enter; installed physical parameters do not enter (outputs are bit-identical with or without a set).  Argument
 * checks -> -1: NULL q; K out of range, a link index out of [-1, n_links), or NULL links / local with K > 0; no output or no cotangent;
 * m < 1 or every tangent NULL; no cotangent output.
 *   device: q [n_q][n_stride], qd and qdd [n_qd][n_stride] fp32 as tds_b200_step_device; J [6K * n_qd][n_stride], vel [6K][n_stride],
 *           acc [6K][n_stride] fp64.  Asynchronous on `stream`.
 *   host:   q [n][n_q], qd and qdd [n][n_qd] fp64 (rounded to fp32); J [n][K][6][n_qd], vel [n][K][6], acc [n][K][6].  Synchronous.
 * _jvp: the outputs' derivatives along m tangents of q, qd and qdd (each may be NULL: zero, not all), one lane per (environment,
 *   tangent) of the dual-number instance, in chunks as tds_b200_step_jvp_*; NULL outputs are skipped.  Device t_q [n_q * m][n_stride],
 *   t_qd and t_qdd [n_qd * m][n_stride], t_J [6K * n_qd * m][n_stride], t_vel and t_acc [6K * m][n_stride] (entry (r, j) at
 *   (r * m + j) * n_stride + e); host t_q [n][n_q][m], t_qd and t_qdd [n][n_qd][m], t_J [n][6K * n_qd][m], t_vel and t_acc [n][6K][m].
 * _vjp: g_x[c] = <G, d(J | vel | acc)/dx_c> for x = q, qd, qdd, for cotangents G_J, G_vel, G_acc in the outputs' layouts (NULL: zero,
 *   not all): the JVP along the n_q + 2 n_qd identity tangents contracted with G on the device.  Any of g_q, g_qd, g_qdd may be NULL,
 *   not all.  Device g_q [n_q][n_stride], g_qd and g_qdd [n_qd][n_stride] fp64 (asynchronous); host g_q [n][n_q], g_qd and g_qdd
 *   [n][n_qd] (synchronous). */
int tds_b200_point_motion_device(tds_b200_sim* sim, const float* q, const float* qd, const float* qdd, int K, const int* links,
                                 const double* local, double* J, double* vel, double* acc, void* stream);
int tds_b200_point_motion_host(tds_b200_sim* sim, const double* q, const double* qd, const double* qdd, int K, const int* links,
                               const double* local, double* J, double* vel, double* acc);
int tds_b200_point_motion_jvp_device(tds_b200_sim* sim, const float* q, const float* qd, const float* qdd, int K, const int* links,
                                     const double* local, int m, const double* t_q, const double* t_qd, const double* t_qdd, double* t_J,
                                     double* t_vel, double* t_acc, void* stream);
int tds_b200_point_motion_jvp_host(tds_b200_sim* sim, const double* q, const double* qd, const double* qdd, int K, const int* links,
                                   const double* local, int m, const double* t_q, const double* t_qd, const double* t_qdd, double* t_J,
                                   double* t_vel, double* t_acc);
int tds_b200_point_motion_vjp_device(tds_b200_sim* sim, const float* q, const float* qd, const float* qdd, int K, const int* links,
                                     const double* local, const double* G_J, const double* G_vel, const double* G_acc, double* g_q,
                                     double* g_qd, double* g_qdd, void* stream);
int tds_b200_point_motion_vjp_host(tds_b200_sim* sim, const double* q, const double* qd, const double* qdd, int K, const int* links,
                                   const double* local, const double* G_J, const double* G_vel, const double* G_acc, double* g_q,
                                   double* g_qd, double* g_qdd);

/* ---- joint-torque and energy regressors of the inertial parameters (DESIGN.md section 7.19) -----------------------------------------
 * tau = Y(q, qd, qdd) pi exactly, with pi [n_pi], n_pi = tds_b200_param_count(sim) - 2: column j is physical-parameter id j + 2 (friction and
 * restitution do not enter inverse dynamics).  Body b (0 = the floating base, i + 1 = link i): columns 10 b + [m, m c_x, m c_y, m c_z,
 * I_xx, I_xy, I_xz, I_yy, I_yz, I_zz], the barycentric parameters of the body: c the centre of mass in the body frame (the frame of the
 * model's com and inertia), I the inertia about the BODY-FRAME ORIGIN in body axes, I = I_com + m (|c|^2 1 - c c^T).  A fixed base's ten
 * columns are zero.  Link i: column 10 (n_links + 1) + 2 i its joint stiffness, the next its damping, as in the parameter ids.
 *   Y [n_qd x n_pi]: at the fp32-rounded q, qd and qdd (qd or qdd may be NULL, meaning zero: Y(q, qd, 0) is the bias regressor, Y(q, 0, 0)
 *     the gravity regressor), Y pi = tds_b200_inverse_dynamics_* at the same inputs (floating base: rows 0..5 the base wrench in the base
 *     frame); the stiffness columns hold q (the axis-angle vector of a spherical joint), the damping columns qd.
 *   yT [n_pi]: the kinetic energy T = yT . pi = sum_b 1/2 v_b^T I_b v_b = 1/2 qd^T M qd with M of tds_b200_mass_matrix_*.
 *   yV [n_pi]: the potential energy V = yV . pi = -sum_b g . (m_b x_com,b) (world coordinates) + 1/2 k q^2 (1/2 k |axis-angle|^2 for a
 *     spherical joint); the damping columns are zero.
 * All fp64; installed physical parameters do not enter (the outputs are bit-identical with or without a set); every entry of a live
 * environment is written, zeros included.  tds_b200.model.inertial_parameters gives pi of the model or of a parameter set.  Argument
 * checks -> -1: NULL q; no output or no cotangent; m < 1 or every tangent NULL; no cotangent output.
 *   device: q [n_q][n_stride], qd and qdd [n_qd][n_stride] fp32 as tds_b200_step_device; Y [n_qd * n_pi][n_stride] (entry (r, c) at row
 *           r * n_pi + c), yT and yV [n_pi][n_stride] fp64.  Asynchronous on `stream`.
 *   host:   q [n][n_q], qd and qdd [n][n_qd] fp64 (rounded to fp32); Y [n][n_qd][n_pi], yT and yV [n][n_pi].  Synchronous.
 * _jvp: the outputs' derivatives along m tangents of q, qd and qdd (each may be NULL: zero, not all), one lane per (environment, tangent)
 *   of the dual-number instance, in chunks as tds_b200_step_jvp_*; NULL outputs are skipped.  Device t_q [n_q * m][n_stride], t_qd and
 *   t_qdd [n_qd * m][n_stride], t_Y [n_qd * n_pi * m][n_stride], t_yT and t_yV [n_pi * m][n_stride] (entry (r, j) at (r * m + j) *
 *   n_stride + e); host t_q [n][n_q][m], t_qd and t_qdd [n][n_qd][m], t_Y [n][n_qd * n_pi][m], t_yT and t_yV [n][n_pi][m].
 * _vjp: g_x[c] = <G, d(Y | yT | yV)/dx_c> for x = q, qd, qdd, for cotangents G_Y, G_yT, G_yV in the outputs' layouts (NULL: zero, not
 *   all): the JVP along the n_q + 2 n_qd identity tangents contracted with G on the device, in chunks of directions within 1 GB.  Any of
 *   g_q, g_qd, g_qdd may be NULL, not all.  Device g_q [n_q][n_stride], g_qd and g_qdd [n_qd][n_stride] fp64 (asynchronous); host g_q
 *   [n][n_q], g_qd and g_qdd [n][n_qd] (synchronous). */
int tds_b200_regressor_device(tds_b200_sim* sim, const float* q, const float* qd, const float* qdd, double* Y, double* yT, double* yV,
                              void* stream);
int tds_b200_regressor_host(tds_b200_sim* sim, const double* q, const double* qd, const double* qdd, double* Y, double* yT, double* yV);
int tds_b200_regressor_jvp_device(tds_b200_sim* sim, const float* q, const float* qd, const float* qdd, int m, const double* t_q,
                                  const double* t_qd, const double* t_qdd, double* t_Y, double* t_yT, double* t_yV, void* stream);
int tds_b200_regressor_jvp_host(tds_b200_sim* sim, const double* q, const double* qd, const double* qdd, int m, const double* t_q,
                                const double* t_qd, const double* t_qdd, double* t_Y, double* t_yT, double* t_yV);
int tds_b200_regressor_vjp_device(tds_b200_sim* sim, const float* q, const float* qd, const float* qdd, const double* G_Y,
                                  const double* G_yT, const double* G_yV, double* g_q, double* g_qd, double* g_qdd, void* stream);
int tds_b200_regressor_vjp_host(tds_b200_sim* sim, const double* q, const double* qd, const double* qdd, const double* G_Y,
                                const double* G_yT, const double* G_yV, double* g_q, double* g_qd, double* g_qdd);

/* ---- inverse mass matrix M^-1(q) and operational-space inverse inertia J M^-1 J^T (DESIGN.md section 7.20) ------------------------
 * Minv [n_qd x n_qd]: the inverse of exactly the matrix tds_b200_mass_matrix_* returns (the CRBA M at the fp32-rounded q, fp64, with the
 *   installed masses, centres of mass and inertias; stiffness, damping, friction and restitution do not enter), by the blocked Cholesky
 *   factor the contact solve uses.  Both triangles, bitwise symmetric (each off-diagonal entry is computed once and written twice).  A
 *   world of several multibodies gives the block-diagonal inverse, with exact zeros between multibodies.  For a floating base this is
 *   NOT the derivative dqdd/dtau of the forward-dynamics step: the reference's floating-base forward dynamics does not invert its own M.
 * Linv [6K x 6K]: the operational-space inverse inertia J M^-1 J^T of a point table of 1 <= K <= TDS_B200_MAX_OSIM_POINTS points (links /
 *   local as in tds_b200_point_motion_*, host memory, passed with each call), with J the 6-row spatial point Jacobian of
 *   tds_b200_point_motion_* (rows [w; x'], floating-base columns in the coordinates of M): entry (6k + r, 6l + s) at row (6k + r) 6K + 6l + s.
 *   Symmetric (one sum per pair, written twice) and positive semi-definite; rank-deficient where a point's chain has fewer than 6 dofs,
 *   so Lambda itself is left to the caller.
 * Either output may be NULL, not both; K is ignored (0 allowed) when Linv and its tangents and cotangents are NULL.  Argument checks ->
 * -1: NULL q; no output (tangent, cotangent); K out of range, a link index out of range, NULL links / local with K > 0, Linv with K = 0;
 * m < 1 or both tangents NULL; no gradient output.  -> -4: t_par / g_par without an installed set.
 *   device: q [n_q][n_stride] fp32 as tds_b200_step_device; Minv [n_qd * n_qd][n_stride], Linv [36 K^2][n_stride] fp64.  Asynchronous.
 *   host:   q [n][n_q] fp64 (rounded to fp32); Minv [n][n_qd][n_qd], Linv [n][6K][6K].  Synchronous.
 * _jvp: the derivatives along m tangents t_q of q and t_par of the installed parameters (either may be NULL: zero), one lane per
 *   (environment, tangent) of the dual-number instance, in chunks as tds_b200_step_jvp_* (dMinv = -Minv dM Minv); Minv and Linv (may be
 *   NULL) receive the values.  Device t_q [n_q * m][n_stride], t_par [k * m][n_stride], t_Minv [n_qd^2 * m][n_stride], t_Linv
 *   [36 K^2 * m][n_stride] (entry (r, j) at (r * m + j) * n_stride + e); host t_q [n][n_q][m], t_par [n][k][m], t_Minv [n][n_qd^2][m],
 *   t_Linv [n][36 K^2][m].
 * _vjp: g_q[c] = <G_Minv, dMinv/dq_c> + <G_Linv, dLinv/dq_c> and, while a set is installed, g_par likewise, for cotangents in the
 *   outputs' layouts (NULL: zero, not both): the JVP along the n_q (+ k) identity tangents contracted with G on the device.  g_q or g_par
 *   may be NULL, not both.  Device g_q [n_q][n_stride], g_par [k][n_stride] fp64 (asynchronous); host g_q [n][n_q], g_par [n][k]. */
#define TDS_B200_MAX_OSIM_POINTS 16
int tds_b200_mass_inverse_device(tds_b200_sim* sim, const float* q, int K, const int* links, const double* local, double* Minv, double* Linv,
                                 void* stream);
int tds_b200_mass_inverse_host(tds_b200_sim* sim, const double* q, int K, const int* links, const double* local, double* Minv, double* Linv);
int tds_b200_mass_inverse_jvp_device(tds_b200_sim* sim, const float* q, int K, const int* links, const double* local, int m, const double* t_q,
                                     const double* t_par, double* Minv, double* Linv, double* t_Minv, double* t_Linv, void* stream);
int tds_b200_mass_inverse_jvp_host(tds_b200_sim* sim, const double* q, int K, const int* links, const double* local, int m, const double* t_q,
                                   const double* t_par, double* Minv, double* Linv, double* t_Minv, double* t_Linv);
int tds_b200_mass_inverse_vjp_device(tds_b200_sim* sim, const float* q, int K, const int* links, const double* local, const double* G_Minv,
                                     const double* G_Linv, double* g_q, double* g_par, void* stream);
int tds_b200_mass_inverse_vjp_host(tds_b200_sim* sim, const double* q, int K, const int* links, const double* local, const double* G_Minv,
                                   const double* G_Linv, double* g_q, double* g_par);

/* ---- point-constrained forward dynamics qdd, f = FD_c(q, qd, tau) (DESIGN.md section 7.21) ----------------------------------------------
 * At the fp32-rounded q, qd and tau (qd or tau may be NULL, meaning zero; tau has one row per dof, a floating base's rows 0..5 being an
 * applied wrench on the base in the base frame as in tds_b200_inverse_dynamics_*, zero for an unactuated base), for a point table of
 * 0 <= K <= TDS_B200_MAX_OSIM_POINTS points (links / local as in tds_b200_point_motion_*, host memory) each held in dims = 3 rows (its
 * linear rows: a point contact that neither slips nor lifts off) or dims = 6 rows (all: a welded frame), with a damping eps >= 0 (finite):
 * with M, h and J, J' qd exactly what tds_b200_mass_matrix_*, tds_b200_inverse_dynamics_*(q, qd, NULL) and tds_b200_point_motion_*(q, qd,
 * NULL) (its J and acc) return at the same inputs and installed parameters, and J_c, d_c their constrained rows (rows 6k + 3 .. 6k + 5
 * of point k for dims 3, all six for dims 6), the KKT system
 *     M qdd - J_c^T f = tau - h,      J_c qdd = -d_c - eps f
 * solved as f = -(J_c M^-1 J_c^T + eps I)^-1 (J_c M^-1 (tau - h) + d_c), qdd = M^-1 (tau - h + J_c^T f), in fp64:
 *   qdd [n_qd]; f [dims K]: per point the force (dims 3) or the wrench [n; f] (dims 6) the constraint applies to the robot at the point, in
 *   world axes (the convention of tds_b200_step_wrench_*'s W: its generalised force is J_c^T f), component r of point k at row dims k + r.
 * K = 0 is the unconstrained forward dynamics qdd = M^-1 (tau - h) in the coordinates of M, so tds_b200_inverse_dynamics_*(q, qd, qdd) =
 * tau on every base; on fixed bases (worlds of several multibodies included) it is the MODE_FD step's qdd, h carrying the stiffness and
 * damping terms.  For a floating base it is not the MODE_FD step's qdd (the reference's floating-base forward dynamics does not invert its
 * own M).  A world of several multibodies is supported: a point constrains only its own multibody's dofs.  If a pivot of the Cholesky
 * factor of J_c M^-1 J_c^T + eps I is <= 0 (a structurally rank-deficient table at eps = 0, e.g. a 3-row point on a planar chain), that
 * environment's outputs are NaN and the others are unaffected; near-singular tables are the caller's to regularise with eps.
 * Either output may be NULL, not both.  Argument checks -> -1: NULL q; no output (tangent output, cotangent); K out of range, a link
 * index out of range, NULL links / local with K > 0; dims not 3 or 6; damping negative or not finite; f (t_f, G_f) with K = 0; m < 1 or
 * every tangent NULL; no gradient output.  -> -4: t_par / g_par without an installed set.
 *   device: q [n_q][n_stride], qd and tau [n_qd][n_stride] fp32 as tds_b200_step_device; qdd [n_qd][n_stride], f [dims K][n_stride] fp64.
 *           Asynchronous on `stream`.
 *   host:   q [n][n_q], qd and tau [n][n_qd] fp64 (rounded to fp32); qdd [n][n_qd], f [n][K][dims].  Synchronous.
 * _jvp: the derivatives along m tangents of q, qd, tau and the installed parameters (each may be NULL: zero, not all), by the dual-number
 *   instances of the inverse dynamics, mass inverse and point motion and of the solve (which differentiates the factorisation), one lane per
 *   (environment, tangent), in chunks of tangents; qdd and f (may be NULL) receive the values.  Device t_q [n_q * m][n_stride], t_qd and
 *   t_tau [n_qd * m][n_stride], t_par [k * m][n_stride], t_qdd [n_qd * m][n_stride], t_f [dims K m][n_stride] (entry (r, j) at
 *   (r * m + j) * n_stride + e); host t_q [n][n_q][m], t_qd and t_tau [n][n_qd][m], t_par [n][k][m], t_qdd [n][n_qd][m], t_f [n][dims K][m].
 * _vjp: g_x[c] = <G_qdd, dqdd/dx_c> + <G_f, df/dx_c> for x = q, qd, tau and, while a set is installed, the parameters, for cotangents in the
 *   outputs' layouts (NULL: zero, not both): the JVP along the n_q + 2 n_qd (+ k) identity tangents contracted with G on the device.  Any of
 *   g_q, g_qd, g_tau, g_par may be NULL, not all.  Device g_q [n_q][n_stride], g_qd and g_tau [n_qd][n_stride], g_par [k][n_stride] fp64
 *   (asynchronous); host g_q [n][n_q], g_qd and g_tau [n][n_qd], g_par [n][k] (synchronous). */
int tds_b200_constrained_dynamics_device(tds_b200_sim* sim, const float* q, const float* qd, const float* tau, int K, const int* links,
                                         const double* local, int dims, double damping, double* qdd, double* f, void* stream);
int tds_b200_constrained_dynamics_host(tds_b200_sim* sim, const double* q, const double* qd, const double* tau, int K, const int* links,
                                       const double* local, int dims, double damping, double* qdd, double* f);
int tds_b200_constrained_dynamics_jvp_device(tds_b200_sim* sim, const float* q, const float* qd, const float* tau, int K, const int* links,
                                             const double* local, int dims, double damping, int m, const double* t_q, const double* t_qd,
                                             const double* t_tau, const double* t_par, double* qdd, double* f, double* t_qdd, double* t_f,
                                             void* stream);
int tds_b200_constrained_dynamics_jvp_host(tds_b200_sim* sim, const double* q, const double* qd, const double* tau, int K, const int* links,
                                           const double* local, int dims, double damping, int m, const double* t_q, const double* t_qd,
                                           const double* t_tau, const double* t_par, double* qdd, double* f, double* t_qdd, double* t_f);
int tds_b200_constrained_dynamics_vjp_device(tds_b200_sim* sim, const float* q, const float* qd, const float* tau, int K, const int* links,
                                             const double* local, int dims, double damping, const double* G_qdd, const double* G_f,
                                             double* g_q, double* g_qd, double* g_tau, double* g_par, void* stream);
int tds_b200_constrained_dynamics_vjp_host(tds_b200_sim* sim, const double* q, const double* qd, const double* tau, int K, const int* links,
                                           const double* local, int dims, double damping, const double* G_qdd, const double* G_f,
                                           double* g_q, double* g_qd, double* g_tau, double* g_par);

/* ---- Coriolis matrix C(q, qd) (DESIGN.md section 7.22) ---------------------------------------------------------------------------------
 * At the fp32-rounded q and qd (qd may be NULL, meaning zero: C = 0), C [n_qd * n_qd] fp64 in the coordinates and layout of
 * tds_b200_mass_matrix (entry (r, c) at r * n_qd + c; a floating base's qd[0:6] is the base-frame twist [w; v]):
 *     C = sum over the bodies i of J_i^T (I_i J_i' + B(I_i, v_i) J_i),  B(I, v) = 1/2 ((v x*) I + bar(I v) - I (v x)),
 *   I_i the spatial inertia of body i (a floating base counts) in world axes about the world origin, J_i its spatial Jacobian in the
 *   coordinates of M (v_i = J_i qd), J_i' its time derivative along qd, bar(f) u = u x* f (Echeandia & Wensing 2021; Pinocchio's
 *   computeCoriolisMatrix).  So C qd = h(q, qd) - h(q, 0) with h the bias forces of tds_b200_inverse_dynamics without joint damping,
 *   C + C^T = M' (the time derivative of M along the motion with velocity qd; M' - 2 C is skew-symmetric), and on coordinates whose rates
 *   are the velocities C is the Christoffel matrix C_ij = sum_k 1/2 (dM_ij/dq_k + dM_ik/dq_j - dM_jk/dq_i) qd_k.  Every entry is written;
 *   a world of several multibodies gives exact zeros between multibodies.
 * While a parameter set is installed, each environment's masses, centres of mass and inertias (links and floating base) are used;
 * stiffness, damping, friction and restitution do not enter.
 * Argument checks: NULL q, no output (C, or t_C for _jvp), no cotangent G, m < 1, every tangent NULL, or no gradient output -> -1; t_par /
 * g_par without an installed set -> -4.
 *   device: q [n_q][n_stride], qd [n_qd][n_stride] fp32; C [n_qd * n_qd][n_stride] fp64.  Asynchronous.
 *   host:   q [n][n_q], qd [n][n_qd] fp64 (rounded to fp32); C [n][n_qd * n_qd].  Synchronous.
 * _jvp: dC along m tangents of q, qd and the installed parameters (each may be NULL: zero, not all); C (may be NULL) receives the value.
 *   Device t_q [n_q * m][n_stride], t_qd [n_qd * m][n_stride], t_par [k * m][n_stride], t_C [n_qd * n_qd * m][n_stride] (entry (r, j) at
 *   (r * m + j) * n_stride + e); host t_q [n][n_q][m], t_qd [n][n_qd][m], t_par [n][k][m], t_C [n][n_qd * n_qd][m].
 * _vjp: g_x[c] = <G, dC/dx_c> for x = q, qd and, while a set is installed, the parameters, for the cotangent G in C's layout: the JVP along
 *   the n_q + n_qd (+ k) identity tangents contracted with G on the device.  Any of g_q, g_qd, g_par may be NULL, not all.  Device g_q
 *   [n_q][n_stride], g_qd [n_qd][n_stride], g_par [k][n_stride] fp64 (asynchronous); host g_q [n][n_q], g_qd [n][n_qd], g_par [n][k]
 *   (synchronous). */
int tds_b200_coriolis_device(tds_b200_sim* sim, const float* q, const float* qd, double* C, void* stream);
int tds_b200_coriolis_host(tds_b200_sim* sim, const double* q, const double* qd, double* C);
int tds_b200_coriolis_jvp_device(tds_b200_sim* sim, const float* q, const float* qd, int m, const double* t_q, const double* t_qd,
                                 const double* t_par, double* C, double* t_C, void* stream);
int tds_b200_coriolis_jvp_host(tds_b200_sim* sim, const double* q, const double* qd, int m, const double* t_q, const double* t_qd,
                               const double* t_par, double* C, double* t_C);
int tds_b200_coriolis_vjp_device(tds_b200_sim* sim, const float* q, const float* qd, const double* G, double* g_q, double* g_qd, double* g_par,
                                 void* stream);
int tds_b200_coriolis_vjp_host(tds_b200_sim* sim, const double* q, const double* qd, const double* G, double* g_q, double* g_qd, double* g_par);

/* ---- derivatives of the inverse dynamics d tau / dq and d tau / dqd (DESIGN.md section 7.23) ----------------------------------------
 * The linearisation of tds_b200_inverse_dynamics at (q, qd, qdd), each [n_qd * n_qd] fp64 per environment, row-major as
 * tds_b200_mass_matrix: row r is tau_r, column c a tangent direction.  d tau / dqdd is M (tds_b200_mass_matrix).  tau is exactly that
 * query's tau: stiffness and damping terms (the spherical joints' axis-angle stiffness included), a floating base's wrench rows in the
 * base frame with gravity rotated into it, and the installed parameter set.  Inputs are rounded to fp32; qd or qdd may be NULL (zero).
 * The columns are in M's coordinates, not q's: column k of d tau / dq is d/de tau(q (+) e e_k) at e = 0, where q (+) e d is the
 * motion with velocity d, whose coordinate rate is dq_dt(q, d) (a floating base: 1/2 q_b (x) (w, 0) and R_b v; a spherical joint: 1/2 q
 * (x) (w, 0); a REVOLUTE_AXIS joint: |axis| d; other joints: d).  So d tau / dq . d equals tds_b200_inverse_dynamics_jvp along
 * t_q = dq_dt(q, d), and the matrices compose with M, C and the point Jacobians.  Every entry is written; a world of several
 * multibodies gives exact zeros between multibodies.
 * Argument checks: NULL q, no output (neither matrix, or neither tangent for _jvp), no cotangent, m < 1, every tangent NULL, or no
 * gradient output -> -1; t_par / g_par without an installed set -> -4.
 *   device: q [n_q][n_stride], qd, qdd [n_qd][n_stride] fp32; dtau_dq, dtau_dqd [n_qd * n_qd][n_stride] fp64 (either may be NULL).
 *           Asynchronous.
 *   host:   q [n][n_q], qd, qdd [n][n_qd] fp64 (rounded to fp32); dtau_dq, dtau_dqd [n][n_qd * n_qd].  Synchronous.
 * _jvp: the tangents of both matrices along m tangents of q (n_q coordinates), qd, qdd and the installed parameters (each may be NULL:
 *   zero, not all), the layout of tds_b200_inverse_dynamics_jvp; dtau_dq, dtau_dqd (may be NULL) receive the values.  Device t_dtau_dq,
 *   t_dtau_dqd [n_qd * n_qd * m][n_stride] (either may be NULL, not both); host [n][n_qd * n_qd][m].
 * _vjp: g_x[c] = <G_dq, d(dtau_dq)/dx_c> + <G_dqd, d(dtau_dqd)/dx_c> for x = q, qd, qdd and, while a set is installed, the parameters
 *   (the JVP along identity tangents contracted on the device).  G_dq or G_dqd may be NULL (zero), not both; any of g_q, g_qd, g_qdd,
 *   g_par may be NULL, not all.  Layouts as tds_b200_inverse_dynamics_vjp. */
int tds_b200_inverse_dynamics_derivatives_device(tds_b200_sim* sim, const float* q, const float* qd, const float* qdd, double* dtau_dq,
                                                 double* dtau_dqd, void* stream);
int tds_b200_inverse_dynamics_derivatives_host(tds_b200_sim* sim, const double* q, const double* qd, const double* qdd, double* dtau_dq,
                                               double* dtau_dqd);
int tds_b200_inverse_dynamics_derivatives_jvp_device(tds_b200_sim* sim, const float* q, const float* qd, const float* qdd, int m,
                                                     const double* t_q, const double* t_qd, const double* t_qdd, const double* t_par,
                                                     double* dtau_dq, double* dtau_dqd, double* t_dtau_dq, double* t_dtau_dqd, void* stream);
int tds_b200_inverse_dynamics_derivatives_jvp_host(tds_b200_sim* sim, const double* q, const double* qd, const double* qdd, int m,
                                                   const double* t_q, const double* t_qd, const double* t_qdd, const double* t_par,
                                                   double* dtau_dq, double* dtau_dqd, double* t_dtau_dq, double* t_dtau_dqd);
int tds_b200_inverse_dynamics_derivatives_vjp_device(tds_b200_sim* sim, const float* q, const float* qd, const float* qdd, const double* G_dq,
                                                     const double* G_dqd, double* g_q, double* g_qd, double* g_qdd, double* g_par,
                                                     void* stream);
int tds_b200_inverse_dynamics_derivatives_vjp_host(tds_b200_sim* sim, const double* q, const double* qd, const double* qdd, const double* G_dq,
                                                   const double* G_dqd, double* g_q, double* g_qd, double* g_qdd, double* g_par);

/* ---- derivatives of the forward dynamics d qdd / dq, d qdd / dqd, d qdd / dtau (DESIGN.md section 7.24) ---------------------------
 * The linearisation of the unconstrained forward dynamics qdd = M^-1 (tau - h) at the fp32-rounded q, qd and tau (qd or tau may be NULL:
 * zero) and the installed parameters, in fp64 per environment:
 *   qdd [n_qd]: tds_b200_constrained_dynamics_* with K = 0, bit for bit;
 *   d qdd / dq [n_qd * n_qd]: -M^-1 d tau / dq, with d tau / dq of tds_b200_inverse_dynamics_derivatives_* taken at (q, qd, qdd) and qdd
 *     read in fp64 (that entry point reads it in fp32);
 *   d qdd / dqd [n_qd * n_qd]: -M^-1 d tau / dqd at the same point;
 *   d qdd / dtau [n_qd * n_qd]: M^-1, tds_b200_mass_inverse_* bit for bit.
 * Row-major as tds_b200_mass_matrix: row r is qdd_r, column c a tangent direction.  The columns are in M's coordinates: column k of
 * d qdd / dq is the derivative along the motion with velocity e_k (see tds_b200_inverse_dynamics_derivatives_*), so d qdd / dq . d equals
 * tds_b200_constrained_dynamics_jvp (K = 0) along t_q = dq_dt(q, d).  The stiffness and damping terms (the spherical joints' axis-angle
 * stiffness included) enter as they enter tds_b200_inverse_dynamics_*.  A floating base's tau rows 0..5 are the applied wrench on the base
 * in the base frame; as for K = 0 of tds_b200_constrained_dynamics_*, qdd is then not the MODE_FD step's qdd (the reference's
 * floating-base forward dynamics does not invert its own M), and these are not that step's derivatives.  A world of several multibodies
 * gives exact zeros between multibodies in all three matrices.  Each output may be NULL, not all four.
 * Argument checks -> -1: NULL q; no output (no tangent output for _jvp, no cotangent for _vjp); m < 1 or every tangent NULL; no gradient
 * output.  -> -4: t_par / g_par without an installed set.
 *   device: q [n_q][n_stride], qd and tau [n_qd][n_stride] fp32; qdd [n_qd][n_stride], the matrices [n_qd * n_qd][n_stride] fp64.
 *           Asynchronous on `stream`.
 *   host:   q [n][n_q], qd and tau [n][n_qd] fp64 (rounded to fp32); qdd [n][n_qd], the matrices [n][n_qd * n_qd].  Synchronous.
 * _jvp: the tangents of the four outputs along m tangents of q (n_q coordinates), qd, tau and the installed parameters (each may be NULL:
 *   zero, not all), second-order terms included, in chunks of tangents; the values (each may be NULL) are written too.  Layouts as
 *   tds_b200_constrained_dynamics_jvp: device t_q [n_q * m][n_stride], t_qd and t_tau [n_qd * m][n_stride], t_par [k * m][n_stride],
 *   t_qdd [n_qd * m][n_stride], t_dqdd_* [n_qd * n_qd * m][n_stride] (entry (r, j) at (r * m + j) * n_stride + e); host [n][dim][m].
 * _vjp: g_x[c] = <G_qdd, dqdd/dx_c> + <G_dq, d(dqdd_dq)/dx_c> + <G_dqd, d(dqdd_dqd)/dx_c> + <G_dtau, d(dqdd_dtau)/dx_c> for x = q, qd, tau
 *   and, while a set is installed, the parameters: the JVP along the n_q + 2 n_qd (+ k) identity tangents contracted on the device.  Each
 *   G may be NULL (zero), not all; any of g_q, g_qd, g_tau, g_par may be NULL, not all.  Layouts as tds_b200_constrained_dynamics_vjp. */
int tds_b200_forward_dynamics_derivatives_device(tds_b200_sim* sim, const float* q, const float* qd, const float* tau, double* qdd,
                                                 double* dqdd_dq, double* dqdd_dqd, double* dqdd_dtau, void* stream);
int tds_b200_forward_dynamics_derivatives_host(tds_b200_sim* sim, const double* q, const double* qd, const double* tau, double* qdd,
                                               double* dqdd_dq, double* dqdd_dqd, double* dqdd_dtau);
int tds_b200_forward_dynamics_derivatives_jvp_device(tds_b200_sim* sim, const float* q, const float* qd, const float* tau, int m,
                                                     const double* t_q, const double* t_qd, const double* t_tau, const double* t_par,
                                                     double* qdd, double* dqdd_dq, double* dqdd_dqd, double* dqdd_dtau, double* t_qdd,
                                                     double* t_dqdd_dq, double* t_dqdd_dqd, double* t_dqdd_dtau, void* stream);
int tds_b200_forward_dynamics_derivatives_jvp_host(tds_b200_sim* sim, const double* q, const double* qd, const double* tau, int m,
                                                   const double* t_q, const double* t_qd, const double* t_tau, const double* t_par,
                                                   double* qdd, double* dqdd_dq, double* dqdd_dqd, double* dqdd_dtau, double* t_qdd,
                                                   double* t_dqdd_dq, double* t_dqdd_dqd, double* t_dqdd_dtau);
int tds_b200_forward_dynamics_derivatives_vjp_device(tds_b200_sim* sim, const float* q, const float* qd, const float* tau, const double* G_qdd,
                                                     const double* G_dq, const double* G_dqd, const double* G_dtau, double* g_q, double* g_qd,
                                                     double* g_tau, double* g_par, void* stream);
int tds_b200_forward_dynamics_derivatives_vjp_host(tds_b200_sim* sim, const double* q, const double* qd, const double* tau, const double* G_qdd,
                                                   const double* G_dq, const double* G_dqd, const double* G_dtau, double* g_q, double* g_qd,
                                                   double* g_tau, double* g_par);

/* ---- the step with its contacts (DESIGN.md section 7.15) -----------------------------------------------------------------
 * One step (MODE_FULL or MODE_WORLD) that also reports what the contact solve did: one record of 10 rows per contact candidate of the
 * model (n_points of tds_b200_get_dims, in the order of tds_b200_contact_pairs and contact_dist), row r of candidate k at row 10 k + r,
 * in world coordinates:
 *   rows 0-2  world_normal_on_b        rows 3-5  world_point_on_b        row 6  distance
 *   rows 7-9  F, the impulse on body B at world_point_on_b (N s; the force is F / dt).  Body A receives -F at the point on A.
 * Rows 0-6 are the reference's ContactPoint fields (contact_point.hpp); the point on A is point_on_b + distance * normal_on_b (plane
 * contacts and contacts between multibodies alike) and is not output.  F = -(p_n n_b + p_1 t_1 + p_2 t_2) with p the solver's row
 * vector of the contact (the PGS result, or the closed-form spring-damper impulse with contact_model 1) and t_1, t_2 the friction
 * directions of the solve (the model's plane_space(-plane normal) for plane contacts, plane_space(normal) between multibodies, as the
 * reference evaluates it: not unit vectors in general, so recover p from F with these directions, not by projection).  A
 * candidate outside the active set (distance >= 0, beyond the solver's contact cap) has F = 0; a candidate between multibodies whose
 * contact function emitted no point has distance +inf and zeros elsewhere.  In a world of several multibodies each contact between
 * multibodies reports the impulse of its own pair's solve.
 * The step always runs on the generic world-frame kernel at the simulator's precision, with the installed parameters if any: q' and qd'
 * are bitwise those of tds_b200_step_device on that kernel (TDS_B200_KERNEL=world).  Arguments as tds_b200_step_device / _host, without
 * qdd_out, reward, done, contact_dist and link_xf.
 *   device: contacts [10 n_points][n_stride] fp32 (asynchronous).  host: contacts [n][n_points][10] fp64; q_out, qd_out may be NULL.
 * _jvp (MODE_FULL): as tds_b200_step_jvp_*, with the output rows q' | qd' | records (n_q + n_qd + 10 n_points).
 * _vjp (MODE_FULL): g_in = g_out^T d(q' | qd' | records) / d(the step's inputs) [cols] and, while a set is installed and g_par is not
 *   NULL, the parameters' cotangents [k], by the JVP along identity tangents.  g_in or g_par may be NULL, not both.  Device g_out
 *   [rows][n_stride], g_in [cols][n_stride], g_par [k][n_stride] fp64 (asynchronous); host g_out [n][rows], g_in [n][cols], g_par [n][k].
 * Returns -1 (bad argument), -2 (mode), -3 (use_pd without tds_b200_set_env), -4 (t_par / g_par without installed parameters). */
int tds_b200_step_contacts_device(tds_b200_sim* sim, int mode, int use_pd, const float* q_in, const float* qd_in, const float* tau_or_action,
                                  float* q_out, float* qd_out, float* contacts, void* stream);
int tds_b200_step_contacts_host(tds_b200_sim* sim, int mode, int use_pd, const double* q, const double* qd, const double* tau_or_action,
                                double* q_out, double* qd_out, double* contacts);
int tds_b200_step_contacts_jvp_device(tds_b200_sim* sim, int mode, int use_pd, const float* q, const float* qd, const float* tau_or_action,
                                      int m, const double* t_in, const double* t_par, double* t_out, void* stream);
int tds_b200_step_contacts_jvp_host(tds_b200_sim* sim, int mode, int use_pd, const double* q, const double* qd, const double* tau_or_action,
                                    int m, const double* t_in, const double* t_par, double* t_out);
int tds_b200_step_contacts_vjp_device(tds_b200_sim* sim, int mode, int use_pd, const float* q, const float* qd, const float* tau_or_action,
                                      const double* g_out, double* g_in, double* g_par, void* stream);
int tds_b200_step_contacts_vjp_host(tds_b200_sim* sim, int mode, int use_pd, const double* q, const double* qd, const double* tau_or_action,
                                    const double* g_out, double* g_in, double* g_par);

/* ---- the step with external wrenches (DESIGN.md section 7.18) ----------------------------------------------------------------------
 * One step (MODE_FD, MODE_NOCONTACT or MODE_FULL) with a wrench W_k = [n_k; f_k] in world axes at every point of a point table: the
 * force f_k acts along a line through the point's world position x_k(q), n_k is a pure moment.  The table is that of the kinematics
 * (0 <= K <= TDS_B200_MAX_KIN_POINTS, point k on links[k] (-1: the base) at local[3k .. 3k+2] in that link's frame, host memory); every
 * environment has its own wrenches.  The generalised force of W_k is J_k^T W_k with J_k the 6-row point Jacobian of
 * tds_b200_point_motion_* at the same q and point (w . n + x' . f is the power).  In the step the wrenches act as the reference's f_ext:
 * each enters the articulated-body bias force of the body it acts on (pA = v x* I v - f_ext, kinematics.hpp:132; a point on a floating
 * base enters the base's bias force), so it reaches qdd through the forward dynamics and q', qd' through the integration and, in
 * MODE_FULL, the contact solve.  A wrench on a fixed base does nothing; in a world of several multibodies a wrench moves only its own
 * multibody.  Gravity, stiffness, damping, PD and installed parameters act as in the step without wrenches, and K = 0 is that step.
 * Inverse dynamics with wrenches is tds_b200_inverse_dynamics_* minus sum_k J_k^T W_k.
 * The step always runs on the generic world-frame kernel at the simulator's precision, with the installed parameters if any.  In the
 * mixed precision the wrenches enter the fp32 forward dynamics as tau does.
 *   device: W [6K][n_stride] fp32 (row 6k + r: component r of [n; f] of point k), q_out, qd_out [dim][n_stride] (MODE_NOCONTACT,
 *   MODE_FULL) or qdd_out [n_qd][n_stride] (MODE_FD), the others may be NULL; asynchronous.
 *   host: W [n][K][6] fp64 (rounded to fp32), outputs [n][dim] fp64.
 * _jvp: as tds_b200_step_jvp_*, rows q' | qd' (qdd in MODE_FD) and columns the step's (tds_b200_jacobian_dims), with the wrenches' tangents
 *   t_W as a block of their own: device t_W [6K * m][n_stride] (row (6k + r) * m + j), host t_W [n][K][6][m].  t_in, t_W and t_par may be
 *   NULL (zero), not all three.
 * _vjp: g_in [cols], g_W (device [6K][n_stride], host [n][K][6]) and, while a set is installed and g_par is not NULL, the parameters'
 *   cotangents g_par [k] = g_out^T d(outputs) / d(inputs), by the JVP along identity tangents (the wrench directions follow the step's
 *   columns and precede the parameters).  g_in, g_W, g_par may be NULL, not all three.  Layouts as tds_b200_step_contacts_vjp_*.
 * Returns -1 (bad argument: a NULL required pointer, K or a link index out of range, m < 1, every tangent or cotangent NULL), -2 (MODE_WORLD),
 * -3 (use_pd without tds_b200_set_env), -4 (t_par / g_par without installed parameters). */
int tds_b200_step_wrench_device(tds_b200_sim* sim, int mode, int use_pd, const float* q_in, const float* qd_in, const float* tau_or_action,
                                int K, const int* links, const double* local, const float* W, float* q_out, float* qd_out, float* qdd_out,
                                void* stream);
int tds_b200_step_wrench_host(tds_b200_sim* sim, int mode, int use_pd, const double* q, const double* qd, const double* tau_or_action, int K,
                              const int* links, const double* local, const double* W, double* q_out, double* qd_out, double* qdd_out);
int tds_b200_step_wrench_jvp_device(tds_b200_sim* sim, int mode, int use_pd, const float* q, const float* qd, const float* tau_or_action,
                                    int K, const int* links, const double* local, const float* W, int m, const double* t_in,
                                    const double* t_W, const double* t_par, double* t_out, void* stream);
int tds_b200_step_wrench_jvp_host(tds_b200_sim* sim, int mode, int use_pd, const double* q, const double* qd, const double* tau_or_action,
                                  int K, const int* links, const double* local, const double* W, int m, const double* t_in, const double* t_W,
                                  const double* t_par, double* t_out);
int tds_b200_step_wrench_vjp_device(tds_b200_sim* sim, int mode, int use_pd, const float* q, const float* qd, const float* tau_or_action,
                                    int K, const int* links, const double* local, const float* W, const double* g_out, double* g_in,
                                    double* g_W, double* g_par, void* stream);
int tds_b200_step_wrench_vjp_host(tds_b200_sim* sim, int mode, int use_pd, const double* q, const double* qd, const double* tau_or_action,
                                  int K, const int* links, const double* local, const double* W, const double* g_out, double* g_in,
                                  double* g_W, double* g_par);

/* Stand-alone integration stages of the fine-grained surface (device SoA arrays as above):
 * integrate_euler (src/dynamics/integrator.hpp:10-133): qd += qdd dt (qdd may be NULL = zero), q += qd dt, floating base
 * quaternion increment + normalisation; integrate_euler_qdd (:141-195): qd += qdd dt only. */
int tds_b200_integrate_euler_device(tds_b200_sim* sim, float* q, float* qd, const float* qdd, void* stream);
int tds_b200_integrate_euler_qdd_device(tds_b200_sim* sim, float* qd, const float* qdd, void* stream);

/* ---- host-buffer path (what VectorizedEnvironment-style callers use) --------------------------------
 * Replaces the per-call loop of SerialForwardStepper / OpenMPForwardStepper::step
 * (examples/ars/ars_vectorized_environment.h:88-137) with MultiBody-style host arrays:
 * q [n_envs][n_q], qd [n_envs][n_qd], tau_or_action [n_envs][n_tau | n_act], AoS fp64 host memory.
 * Copies in, steps once, copies out (synchronous).  Outputs may be NULL. */
int tds_b200_step_host(tds_b200_sim* sim, int mode, int use_pd, const double* q, const double* qd,
                       const double* tau_or_action, double* q_out, double* qd_out, double* qdd_out,
                       double* contact_dist);

/* Environment-level step on the sim's own resident state: VectorizedEnvironment::step
 * (examples/ars/ars_vectorized_environment.h:214-291) minus the policy: actions [n_envs][n_act] fp32
 * host (pinned for speed) -> obs [n_envs][n_q+n_qd], rewards [n_envs], dones [n_envs] fp32 host.
 * State stays on the device between calls.  Synchronous.
 * Fast paths (same results): with pinned (mapped) buffers and a model the library holds a specialised kernel for, the
 * step kernel itself reads the actions from and writes obs / rewards / dones to host memory (one launch, no copies);
 * otherwise pinned buffers -> the copy/transpose/step/pack/copy sequence is replayed from a CUDA graph captured on the
 * third call with the same pointers, and obs, rewards, dones adjacent in memory (rewards == obs + n_envs*(n_q+n_qd),
 * dones == rewards + n_envs) -> one device->host copy instead of three. */
/* ---- contact-pair index lists (World::compute_contacts_multi_body_internal, src/world.hpp:212-281;
 * MultiBodyContactPoint::{multi_body_a, link_a, multi_body_b, link_b}, src/mb_constraint_solver.hpp:29-40) -------------
 * The candidate points of a model are static: plane (body 0, base link -1) x every sphere / capsule end of the robot
 * (body 1) in the reference's enumeration order.  tds_b200_contact_pairs writes one tuple (body_a, link_a, body_b, link_b)
 * per candidate (the list World::mb_contacts_ holds after every step) and returns their number.
 * tds_b200_contact_list_*: the list the constraint solver keeps in a step (all candidates with keep_all_points, else
 * those with distance < 0: resolve_collision, mb_constraint_solver.hpp:169-180), computed on the device from the
 * contact distances of that step: count[e] and (link_a, link_b) of the k-th kept point, -9 beyond count.
 *   device: contact_dist [n_points][ns] (output of tds_b200_step_device), count [ns], links [2 * n_points][ns]
 *   host:   uses the distances of the last tds_b200_step_host(..., contact_dist != NULL); count [n], links [n][n_points][2]
 * Worlds of several multibodies (TDSM_H_NBODIES > 1, include/tds_b200_model.h): the multibodies of the model are bodies
 * 1, 2, ... of the world (the plane, if any, is body 0), link indices are those inside their multibody, and the candidates
 * BETWEEN multibodies (sphere-sphere, capsule-sphere; one list of World::mb_contacts_ per pair a < b, src/world.hpp:212-281)
 * follow the plane candidates; contact_dist carries their distances in the same order (+inf: the contact function emitted no
 * point).  tds_b200_contact_list_candidates_host: cand [n][n_points] = index into the candidate list of the k-th kept point. */
int tds_b200_contact_pairs(const tds_b200_sim* sim, int* tuples, int cap);
int tds_b200_model_contact_pairs(const double* model, int n_model, int* tuples, int cap);   /* host-only, from a flat model */
/* (mb_a, link_a, geom_a, mb_b, link_b, geom_b) per candidate = the loop indices of world.hpp:212-240 at which the point is emitted
 * (geom: index in collision_geometries(link)); 6 ints per candidate, same order as tds_b200_contact_pairs */
int tds_b200_contact_tuples(const tds_b200_sim* sim, int* tuples, int cap);
int tds_b200_model_contact_tuples(const double* model, int n_model, int* tuples, int cap);   /* host-only */
int tds_b200_contact_list_device(tds_b200_sim* sim, const float* contact_dist, int* count, int* links, void* stream);
int tds_b200_contact_list_host(tds_b200_sim* sim, int* count, int* links);
int tds_b200_contact_list_candidates_host(tds_b200_sim* sim, int* count, int* cand);

int tds_b200_env_set_state_host(tds_b200_sim* sim, const double* q, const double* qd);
int tds_b200_env_get_state_host(tds_b200_sim* sim, double* q, double* qd);
int tds_b200_env_step_host(tds_b200_sim* sim, const float* actions, float* obs, float* rewards, float* dones);
/* Same, device-resident: actions/reward/done are device SoA arrays; advances the resident state. */
int tds_b200_env_step_device(tds_b200_sim* sim, const float* actions, float* reward, float* done, void* stream);
/* Device pointers of the resident state (SoA fp32 [n_q][ns], [n_qd][ns]). */
/* ---- environment layer on the device (what surrounds the step in the reference's ARS loop) ---------------------
 * Episode reset, LaikagoContactSimulation::reset (examples/environments/laikago_environment2.h:63-116): environments with
 * mask[e] != 0 (all when mask is NULL) are set to the reset pose of tds_b200_set_auto_reset plus noise on the actuated
 * joints (noise: device [n_act][n_stride], or NULL -> U(-noise_amp, noise_amp) from a counter-based generator keyed by
 * (seed, env, joint); the reference draws std::rand() * 0.05), qd = 0, then settle_steps env-steps with zero actions;
 * the other environments keep their state. */
int tds_b200_env_reset_device(tds_b200_sim* sim, const float* mask, const float* noise, float noise_amp,
                              unsigned long long seed, int settle_steps, void* stream);
/* rollout_length steps of ARSVectorizedWorker::rollouts (examples/ars/ars_vectorized_worker.h:51-141) without leaving
 * the GPU: per environment a linear policy with bias (VectorizedEnvironment::policy, ars_vectorized_environment.h:293-300;
 * parameters = weights [n_act][n_q+n_qd] row-major | biases [n_act], device layout [n_params][n_stride]) on the observation
 * (q | qd, x and y zeroed), the env-step, sticky done; total_rewards[e] = sum of (reward - shift) and steps[e] over the
 * steps the environment was alive.  Device pointers; asynchronous on `stream` (NULL: the simulator's own stream, the one
 * the host-buffer entry points use; the same holds for tds_b200_env_reset_device). */
int tds_b200_env_rollout_device(tds_b200_sim* sim, const float* policy, int n_params, int rollout_length, float shift,
                                float* total_rewards, int* steps, void* stream);
/* Observation-filter statistics of the rollouts (ars_vectorized_worker.h:93-110, running_stat.h): with a non-NULL buffer
 * (device, [3 * (n_q + n_qd)][n_stride] = count | mean | S per component, caller-owned, zero to clear) every rollout step
 * pushes the observation the policy saw into a per-environment Welford accumulator.  NULL switches it off. */
int tds_b200_env_set_obs_stats(tds_b200_sim* sim, float* stats);
/* ARS on the device (ARSVectorizedWorker::do_rollouts, ars_vectorized_worker.h:205-262; ARSLearner::weighted_sum_custom and
 * train_step, ars_learner.h:67-91,185-189).  w [n_params] device; deltas [n_params][n_stride] unit normals, one direction
 * per environment; perturb: params[p][e] = w[p] + scale * deltas[p][e] (scale = +-delta_std) in the rollout layout;
 * update: w[p] += step_size * delta_std / n * sum_e (r_pos[e] - r_neg[e]) * deltas[p][e]. */
int tds_b200_ars_perturb_device(tds_b200_sim* sim, const float* w, const float* deltas, float scale, float* params, int n_params,
                                void* stream);
int tds_b200_ars_update_device(tds_b200_sim* sim, float* w, const float* deltas, const float* r_pos, const float* r_neg,
                               float delta_std, float step_size, int n_params, void* stream);
/* reset + rollout with host buffers: policy [n_envs][n_params], noise [n_envs][n_act] or NULL, results to host. */
int tds_b200_env_rollout_host(tds_b200_sim* sim, const double* policy, int n_params, int rollout_length, double shift,
                              const double* noise, double noise_amp, unsigned long long seed, int settle_steps,
                              double* total_rewards, int* steps);

/* Env step + visual-transform stream in the instancing renderer's layout (instance = env * n_visuals + v):
 * positions[4 i] = x, y, z, 1 and orientations[4 i] = quaternion xyzw (device float arrays of 4 * n_envs * n_visuals),
 * the two arrays TinyGLInstancingRenderer holds (src/visualizer/opengl/tiny_gl_instancing_renderer.cpp:366-367,440-457);
 * same per-visual transforms as the records of the v1 output (locomotion_contact_simulation.h:281-299). */
int tds_b200_num_visuals(const tds_b200_sim* sim);
int tds_b200_env_step_visual_device(tds_b200_sim* sim, const float* actions, float* reward, float* done, float* positions,
                                    float* orientations, void* stream);

/* The simulator's own (non-blocking) cudaStream_t: what the host-buffer entry points and the env-layer calls with a NULL
 * stream run on.  Work enqueued by the caller on other streams is NOT ordered against it. */
void* tds_b200_stream(tds_b200_sim* sim);
float* tds_b200_env_q(tds_b200_sim* sim);
float* tds_b200_env_qd(tds_b200_sim* sim);

/* ---- C-ABI v1 drop-in ---------------------------------------------------------------------------------
 * Exactly the symbols the reference's CudaSourceGen emits and ars_train_policy_cuda / cuda_codegen dlsym
 * (src/utils/cuda_codegen.hpp:156-266; loaded at examples/ars/ars_train_policy_cuda.cpp:183-230):
 *   input  = num_total_threads blocks of input_dim  (51 = q18|qd18|action12|kp,kd,max_force) fp64, AoS, host
 *   output = num_total_threads blocks of output_dim (411 = q18|qd18|17x(pos3,quat4)|up.z|zeros) fp64, AoS, host
 * Synchronous: H2D, one step, D2H.  num_blocks / num_threads_per_block are accepted and ignored (the
 * launch geometry is chosen for sm_90a). */
typedef struct {
  int output_dim;
  int input_dim;
  int global_dim;
} CudaFunctionMetaData; /* src/utils/cuda_codegen.hpp:27-31 */

void cuda_model_laikago_forward_zero(int num_total_threads, int num_blocks, int num_threads_per_block,
                                     double* output, const double* input);
CudaFunctionMetaData cuda_model_laikago_forward_zero_meta(void);
void cuda_model_laikago_forward_zero_allocate(int num_total_threads);
void cuda_model_laikago_forward_zero_deallocate(void);
/* "cuda_model_" + AntContactSimulation2::env_name() (examples/ars/ars_train_policy_cuda.cpp:507, ant_environment2.h):
 * input_dim 39 = q14|qd14|action8|kp,kd,max_force, output_dim 155 = q14|qd14|9x(pos3,quat4)|up.z|zeros */
void cuda_model_ant_forward_zero(int num_total_threads, int num_blocks, int num_threads_per_block,
                                 double* output, const double* input);
CudaFunctionMetaData cuda_model_ant_forward_zero_meta(void);
void cuda_model_ant_forward_zero_allocate(int num_total_threads);
void cuda_model_ant_forward_zero_deallocate(void);

/* ---- C-ABI v2 (alt): what tds::CudaLibrary / CudaModel / CudaFunction load (src/utils/cuda/cuda_library.hpp:51-68,
 * cuda_model.hpp:14-25, cuda_function.hpp:78-100; emitted at src/utils/cuda/cuda_codegen.hpp:32-231).  One model,
 * "b200_laikago" (same 51 -> 411 function as cuda_model_laikago) with its <model>_jacobian. */
typedef struct { int output_dim; int local_input_dim; int global_input_dim; bool accumulated_output; } CudaFunctionMetaDataV2;
void model_info(char const* const** names, int* count);
CudaFunctionMetaDataV2 b200_laikago_forward_zero_meta(void);
void b200_laikago_forward_zero_allocate(int num_total_threads);
void b200_laikago_forward_zero_deallocate(void);
bool b200_laikago_forward_zero_send_local(int num_total_threads, const double* input);
bool b200_laikago_forward_zero_send_global(const double* input);
void b200_laikago_forward_zero(int num_total_threads, int num_blocks, int num_threads_per_block, double* output);
/* <model>_jacobian of the same generation (src/utils/cuda/cuda_codegen.hpp:303-426): rows = the 36 state outputs q' | qd'
 * (output sparsity, :283-288), columns = the 51 local inputs; output_dim = 36 * 51 per thread, row-major, not accumulated. */
CudaFunctionMetaDataV2 b200_laikago_jacobian_meta(void);
void b200_laikago_jacobian_allocate(int num_total_threads);
void b200_laikago_jacobian_deallocate(void);
bool b200_laikago_jacobian_send_local(int num_total_threads, const double* input);
bool b200_laikago_jacobian_send_global(const double* input);
void b200_laikago_jacobian(int num_total_threads, int num_blocks, int num_threads_per_block, double* output);

/* ---- the RigidBody path of World::step (src/world.hpp:293-363, src/rigid_body.hpp, src/rb_constraint_solver.hpp) ----------
 * A world of up to 16 rigid bodies with ONE collision shape each (sphere, plane, capsule, box), a batch of such worlds per
 * simulator, one GPU lane per world: apply_gravity / apply_force_impulse / clear_forces, contacts of every pair through the
 * reference's dispatcher (sphere-sphere, plane-sphere / capsule / box, capsule-sphere, and the swapped calls), the
 * sequential-impulse solver (num_solver_iterations sweeps over the contact list), integrate.
 *   desc   [n_bodies][6]  = mass (0: static), shape (TDSG_*, tds_b200_model.h), p0..p3: sphere radius | capsule radius, length |
 *                           box extents | plane normal [3], constant
 *   state  per body 13 doubles: position [3], orientation xyzw [4], linear velocity [3], angular velocity [3]
 *          device layout [13 * n_bodies][n_stride] fp64 (n_stride = n_worlds rounded up to 32), host layout [n_worlds][n_bodies][13]
 *   force  RigidBody::apply_central_force before the FIRST step ([3 * n_bodies][n_stride] / [n_worlds][n_bodies][3]) or NULL
 * Defaults are the reference's (dt 1/60 is ours): gravity (0, 0, -9.81), friction 0.5, restitution 0, erp 0.1, 1 solver iteration.
 * tds_b200_rigid_jacobian_host: d state_out / d (state | force) [n_worlds][13 n_bodies][16 n_bodies] by forward-mode dual numbers
 * (python/examples/billiard_optimization.py differentiates exactly this path). */
typedef struct tds_b200_rigid tds_b200_rigid;
tds_b200_rigid* tds_b200_rigid_create(const double* desc, int n_bodies, int n_worlds, int device);
void tds_b200_rigid_destroy(tds_b200_rigid* h);
int tds_b200_rigid_set_params(tds_b200_rigid* h, double dt, const double* gravity, double friction, double restitution, double erp,
                              int num_solver_iterations);
int tds_b200_rigid_step_device(tds_b200_rigid* h, const double* state_in, double* state_out, const double* force, int steps, void* stream);
int tds_b200_rigid_step_host(tds_b200_rigid* h, const double* state, const double* force, int steps, double* state_out);
int tds_b200_rigid_jacobian_host(tds_b200_rigid* h, const double* state, const double* force, int steps, double* state_out, double* jac);
/* Vector-Jacobian product of `steps` World::step calls: (g_state, g_force) = g_state_out^T d state_out / d (state, force), by the
 * taping instance of the rigid-body kernel one step at a time: the forward keeps the steps + 1 states on the device, then steps
 * single-step reverse sweeps run backwards, chaining the state cotangent (the tape never holds more than one step).  The force
 * acts in the first step only.  force may be NULL (zero force); g_force may be NULL.
 *   device: state / g_state_out / g_state [13 n_bodies][n_stride], force / g_force [3 n_bodies][n_stride] fp64
 *   host:   state, g_state_out, g_state [n_worlds][n_bodies][13], force, g_force [n_worlds][n_bodies][3] fp64.  Synchronous. */
int tds_b200_rigid_vjp_device(tds_b200_rigid* h, const double* state, const double* force, int steps, const double* g_state_out,
                              double* g_state, double* g_force, void* stream);
int tds_b200_rigid_vjp_host(tds_b200_rigid* h, const double* state, const double* force, int steps, const double* g_state_out,
                            double* g_state, double* g_force);
/* Jacobian-vector products of `steps` World::step calls: t_state_out = d state_out / d (state | force) along m tangents, by the
 * dual-number kernel seeded with the tangents, one lane per (world, tangent) running the whole rollout in one launch (no
 * checkpoints).  The force acts in the first step only; a force tangent with force NULL differentiates at zero force.  state_out (the
 * rollout's end state, written by the lanes of tangent 0) may be NULL and must not alias state.  t_state or t_force may be NULL
 * (zero tangent), not both; m < 1, m > 65535 or a NULL required pointer -> -1.
 *   device: state [13 n_bodies][n_stride], force [3 n_bodies][n_stride]; t_state / t_state_out [13 n_bodies * m][n_stride],
 *           t_force [3 n_bodies * m][n_stride] fp64, entry (r, j) of world e at (r * m + j) * n_stride + e.  Asynchronous.
 *   host:   state [n_worlds][n_bodies][13], force [n_worlds][n_bodies][3]; t_state / t_state_out [n_worlds][n_bodies][13][m],
 *           t_force [n_worlds][n_bodies][3][m] fp64.  Synchronous. */
int tds_b200_rigid_jvp_device(tds_b200_rigid* h, const double* state, const double* force, int steps, int m, const double* t_state,
                              const double* t_force, double* state_out, double* t_state_out, void* stream);
int tds_b200_rigid_jvp_host(tds_b200_rigid* h, const double* state, const double* force, int steps, int m, const double* t_state,
                            const double* t_force, double* state_out, double* t_state_out);

/* ---- per-world physical parameters of the rigid-body world (DESIGN.md 7.11): system identification and domain randomisation ------
 * Parameter ids, one value per world each:
 *   0            friction (RigidWorld friction, tds_b200_rigid_set_params)
 *   1            restitution
 *   2 + 4 b + c  body b: c = 0 mass; c = 1..3 shape sizes: sphere radius (c = 1); capsule radius, length (c = 1, 2); box extents
 *                x, y, z (c = 1..3).  The box's corner radius stays 1e-2.
 * tds_b200_rigid_param_count: 2 + 4 n_bodies.
 * Refused (-2, reason in tds_b200_last_error): an id out of range, an id given twice, the mass of a static body (model mass 0), a size
 * component the shape does not have, any id of a plane.  A body's static / dynamic status stays that of the description.
 *
 * tds_b200_rigid_set_physical_params_*: install k parameters; the handle copies the values into a buffer it owns (new values for the
 * same ids keep the buffer).  k = 0 clears the set.  device: values [k][n_stride] fp64 device pointer, copied on `stream` (NULL: the
 * world's stream) WITHOUT checking the values.  host: values [n_worlds][k] fp64, synchronous; a non-finite value, a mass or size <= 0,
 * a negative friction or restitution -> -3.  While a set is installed, rigid_step_*, rigid_jacobian_host, rigid_vjp_* and rigid_jvp_*
 * use each world's values for those ids (and the description's for the rest).
 *
 * The derivative entries below return -4 when no set is installed; their other argument checks are those of the entries they extend
 * (-1).  Columns and slots are in the order of the installed ids.
 *   tds_b200_rigid_param_jacobian_host: d state_out / d (installed parameters) of `steps` steps, jac [n_worlds][13 n_bodies][k].
 *   tds_b200_rigid_vjp_params_*: tds_b200_rigid_vjp_* that also writes g_par = g_state_out^T d state_out / d (parameters), summed over
 *     all `steps` (the force still acts in step 0 only): device [k][n_stride], host [n_worlds][k].  g_par must not be NULL.
 *   tds_b200_rigid_jvp_params_*: tds_b200_rigid_jvp_* with parameter tangents t_par: device [k * m][n_stride] (entry (s, j) at
 *     (s * m + j) * n_stride + e), host [n_worlds][k][m].  t_state, t_force and t_par may each be NULL (zero tangent), not all three. */
int tds_b200_rigid_param_count(const tds_b200_rigid* h);
int tds_b200_rigid_set_physical_params_device(tds_b200_rigid* h, int k, const int* ids, const double* values, void* stream);
int tds_b200_rigid_set_physical_params_host(tds_b200_rigid* h, int k, const int* ids, const double* values);
int tds_b200_rigid_param_jacobian_host(tds_b200_rigid* h, const double* state, const double* force, int steps, double* state_out, double* jac);
int tds_b200_rigid_vjp_params_device(tds_b200_rigid* h, const double* state, const double* force, int steps, const double* g_state_out,
                                     double* g_state, double* g_force, double* g_par, void* stream);
int tds_b200_rigid_vjp_params_host(tds_b200_rigid* h, const double* state, const double* force, int steps, const double* g_state_out,
                                   double* g_state, double* g_force, double* g_par);
int tds_b200_rigid_jvp_params_device(tds_b200_rigid* h, const double* state, const double* force, int steps, int m, const double* t_state,
                                     const double* t_force, const double* t_par, double* state_out, double* t_state_out, void* stream);
int tds_b200_rigid_jvp_params_host(tds_b200_rigid* h, const double* state, const double* force, int steps, int m, const double* t_state,
                                   const double* t_force, const double* t_par, double* state_out, double* t_state_out);

#ifdef __cplusplus
}
#endif
#endif /* TDS_B200_H */
