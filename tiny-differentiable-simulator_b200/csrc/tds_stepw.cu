// World-frame batched env-step kernel for sm_90a (successor of tds_step.cu's link-frame kernel).
//
// Same reference path as tds_step.cu (PD -> kinematics -> ABA -> integrate_euler_qdd -> contacts -> CRBA ->
// LCP/PGS -> integrate_euler; citations at each stage), restructured once more around the instruction count,
// because with 4096 environments one warp owns an SM and every instruction is paid at single-warp latency:
//
//   * ALL spatial quantities of an environment live in ONE common frame: world axes, origin O that moves
//     with the robot (base position, or the end of the translation-only root chain).  Then
//       - velocities / accelerations propagate by addition (v_i = v_parent + S_i qd_i),
//       - articulated and composite inertias accumulate by addition: the per-link congruence transform
//         X^T Ia X of the reference (forward_dynamics.hpp:187-189, mass_matrix.hpp:45-46; ~250 FMA per link
//         even in block form) disappears; the price is moving each link's rigid-body inertia into the common
//         frame once (~70 FMA, shared by ABA and CRBA),
//       - M_ij = S_j . (Ic_i S_i) and contact Jacobian columns = S_j.bot + S_j.top x x_c need no chain walks
//         with transforms.
//     Equivalent to the reference in exact arithmetic (spatial algebra is frame invariant); the floating-base
//     quirks that ARE frame dependent (block inverse with C = -H, gyroscopic term, un-rotated gravity) are
//     evaluated in the base frame exactly as the reference does.
//   * Only S (6 numbers), v/c/a, U, 1/D, u per link are kept; world transforms are carried in registers and
//     stored only for branch points.
//   * The contact solve works on 3x3 register blocks (dofs padded to a multiple of 3): blocked Cholesky,
//     blocked forward substitution of 3 right-hand sides per contact, matrix-free PGS on w = Y p, blocked
//     back substitution.  A block op is 18 shared loads for 27 FMA with compile-time indexing.
//   * Scalar types: RA (ABA) fp32, RC (kinematics, contact geometry, inertias in the common frame, CRBA
//     products, Jacobians, LCP right-hand side) fp64, RS (factorisation, substitutions, PGS) fp32 in the
//     default mixed mode.
#include <cuda_runtime.h>

#include "tds_wcommon.cuh"

namespace tdsw {


// per-link region, element offsets: [rigid inertia (10 RC) | later U (6 RA), invD, u] then v / c / a (6 RA)

// kernel argument of the instances without installed physical parameters: nothing
struct NoPar {};
// tangents of the Jacobian-vector product instances (JV, DESIGN.md section 7.10): input column c of tangent j is
// t_in[(c * m + j) * n_stride + e], installed parameter slot s is t_par[(s * m + j) * n_stride + e]; null: zero tangent
struct JvpTan { const double* t_in; const double* t_par; int m; };
struct NoParJvp { JvpTan jv; };
struct ParMapJvp : ParMap { JvpTan jv; };
// kernel argument of the kinematics instances (KIN, DESIGN.md section 7.13): the outputs (each may be null) and the point table, the
// same for every environment: point k sits on link link[k] (-1: the base) at local[3k..3k+2] in that link's frame
struct KinArg {
  double* xf; double* x; double* J;
  int K;
  int link[TDS_MAX_KIN_POINTS];
  double local[3 * TDS_MAX_KIN_POINTS];
};
struct KinArgJvp : KinArg { JvpTan jv; };
// kernel argument of the contact-reporting value instances (CF, DESIGN.md section 7.15): the records [10 * n_pts][ns] fp32.  The JVP
// instances write the records' dual parts into io.jac behind q' | qd' and take the plain JVP arguments.
struct CfArg { float* cf; };
struct CfArgPar : ParMap { float* cf; };
// kernel argument of the centroidal instances (CEN, DESIGN.md section 7.16): the argument of the same instance without CEN and the outputs
template <typename B> struct CenArg : B { double* com; double* A; double* bias; };
// kernel argument of the point-motion instances (MOT, DESIGN.md section 7.17): the point table of KinArg (B = KinArg or KinArgJvp), whose
// J is the 6-row spatial point Jacobian here (xf and x are not read), and the outputs vel and acc
template <typename B> struct MotArg : B { double* vel; double* acc; };
// kernel argument of the external-wrench instances (EXT, DESIGN.md section 7.18): the argument of the same instance without EXT (B = NoPar,
// ParMap, NoParJvp or ParMapJvp) and the point table of KinArg with the wrenches W [6K][ns] fp32 (row 6k + r: component r of [n; f] of
// point k), their tangents t_W [6K * m][ns] (JV instances; null: zero tangent), the arena word x_ext of the per-link wrench sums and the
// links that have points (bit i: link i), the only ones whose sums are stored and read
struct ExtPts {
  const float* W; const double* t_W;
  unsigned long long links_with_points;
  int K, x_ext;
  int link[TDS_MAX_KIN_POINTS];
  double local[3 * TDS_MAX_KIN_POINTS];
};
template <typename B> struct ExtArg : B { ExtPts ext; };
// kernel argument of the regressor instances (REG, DESIGN.md section 7.19): the argument of the same instance without REG (B = NoPar or
// NoParJvp) and the energy regressors' outputs yT and yV (each may be null)
template <typename B> struct RegArg : B { double* yT; double* yV; };
template <bool PAR, bool JV = false, bool KIN = false, bool CF = false, bool CEN = false, bool MOT = false, bool EXT = false,
          bool REG = false> struct ParArg { typedef NoPar type; };
template <> struct ParArg<true, false> { typedef ParMap type; };
template <> struct ParArg<false, true> { typedef NoParJvp type; };
template <> struct ParArg<true, true> { typedef ParMapJvp type; };
template <> struct ParArg<false, false, true> { typedef KinArg type; };
template <> struct ParArg<false, true, true> { typedef KinArgJvp type; };
template <> struct ParArg<false, false, false, true> { typedef CfArg type; };
template <> struct ParArg<true, false, false, true> { typedef CfArgPar type; };
template <> struct ParArg<false, true, false, true> { typedef NoParJvp type; };
template <> struct ParArg<true, true, false, true> { typedef ParMapJvp type; };
template <bool PAR, bool JV> struct ParArg<PAR, JV, false, false, true> { typedef CenArg<typename ParArg<PAR, JV>::type> type; };
template <> struct ParArg<false, false, false, false, false, true> { typedef MotArg<KinArg> type; };
template <> struct ParArg<false, true, false, false, false, true> { typedef MotArg<KinArgJvp> type; };
template <bool PAR, bool JV> struct ParArg<PAR, JV, false, false, false, false, true> { typedef ExtArg<typename ParArg<PAR, JV>::type> type; };
template <bool JV> struct ParArg<false, JV, false, false, false, false, false, true> { typedef RegArg<typename ParArg<false, JV>::type> type; };

// CF, dual instances: the part of a record's dual number they write - the tangent (d).  The host build of the tests also compiles them
// with the value (v), for an fp64 value path of the records that central differences can resolve.
#ifndef TDS_CF_DUAL_PART
#define TDS_CF_DUAL_PART d
#endif

// CF: the (c + 1)-th set bit of mask (the candidate index of active contact c; the active contacts are compacted in candidate order)
TDS_D int cf_nth_bit(unsigned long long mask, int c) {
  for (int i = 0; i < 64; ++i)
    if ((mask >> i) & 1ull) { if (c-- == 0) return i; }
  return -1;
}

// joint stiffness and damping enter the step at fp32, as DevModel stores them; the derivative is taken at the rounded value
TDS_D double f32_round(double x) { return (double)(float)x; }
template <typename T> TDS_D Dual<T> f32_round(Dual<T> x) { x.v = (T)(float)x.v; return x; }
template <typename T> TDS_D Tape<T> f32_round(Tape<T> x) { x.v = (T)(float)x.v; return x; }

// RQ: scalar of the state vectors (q, qd, tau): float, or the dual number type in the differentiable instance
// (RA = RC = RS = RQ = Dual<double>: blockIdx.y + io.jac_dir0 is the input direction of the lane, see tds_dual.cuh),
// or the taping scalar of the vector-Jacobian product (RA = RC = RS = RQ = Tape<double>, one lane per environment: the
// lane records its step and sweeps it backwards from io.g_out at the end, see tds_tape.cuh).
// PAR: per-environment physical parameters (DESIGN.md section 7.9).  Parameter slot s of the lane is pm.values[s * n_stride + e];
// pm also says which model quantity each slot replaces.  In the dual instance slot s is input direction n_in_ad + s, in the taping
// instance leaf n_in_ad + s (after the state / control inputs, so g_in keeps its layout).  The values are read where the model
// values are read (once per step each; the reads of a warp are coalesced), so the arena layout does not change.
// JV (dual instances only): Jacobian-vector product.  The lane's direction is tangent j = blockIdx.y + io.jac_dir0 of pm.jv; every
// input and installed parameter is seeded with its entry of that tangent, and the dual parts of the outputs are column j of io.jac
// (io.jac_n_in = m columns): t_out = J V, row-major per environment as the Jacobian.
// MASS: the joint-space mass matrix M(q) (DESIGN.md section 7.12), launched in MODE_NOCONTACT.  Pass 1 from q alone (qd = 0, no PD, tau or
// contact detection: mass_matrix.hpp:36),
// the CRBA of pass 2 and the floating-base block as if a contact were active, then the dense symmetric n_qd x n_qd matrix in place of
// the solve: entry (r, c) at io.jac[(r * n_qd + c) * ns + e] (fp64 instance), or its dual part as column j of an m-column Jacobian,
// io.jac[((r * n_qd + c) * m + j) * ns + e] (JV instance, t_in = the q tangents).  ABA, integration and reward are not compiled in.
// KIN: forward kinematics and linear point Jacobians (DESIGN.md section 7.13), launched in MODE_NOCONTACT with the point table as pm.
// Pass 1 from q alone (qd = 0, no PD, tau or contact detection: forward_kinematics_q), without the inertias pass 2 needs; as pass 1
// reaches link l it writes l's world transform (pm.xf, the layout of io.link_xf), and the world position p_l + R_l local + O
// (pm.x) and the 3 x n_qd Jacobian (pm.J, jacobian.hpp:13-83) of every point on l.  Returns before pass 2.  Row r of a output at
// out[r * ns + e] (fp64 instance), or its dual part as column j of an m-column Jacobian, out[(r * m + j) * ns + e] (JV instance).
// INV: inverse dynamics tau = ID(q, qd, qdd) by the recursive Newton-Euler algorithm (DESIGN.md section 7.14), launched in MODE_NOCONTACT
// with the simulator's gravity.  qdd arrives in io.tau_in [n_qd][ns] (null: zero; so does a null io.qd_in), tangent input index
// n_q + n_qd + k.  Pass 1 carries the accelerations a_i = a_parent + S_i qdd_i + v_i x (S_i qd_i) along with v (a_base = -g, or the
// floating base's R_b qdd[0:6] - g), forms f_i = r_i a_i + v_i x* (r_i v_i) from the rigid inertia about O and adds S_j . f_i to tau_j
// for i and its moving ancestors j (all in the common frame: no transforms); a branch point's a_i is kept over its rigid-inertia words,
// which nothing else reads.  Then the stiffness and damping terms the ABA subtracts, the floating base's wrench in the base frame, and
// tau [n_qd] at io.jac[r * ns + e] (fp64 instance) or its dual part at io.jac[(r * m + j) * ns + e] (JV instance).  Returns before pass 2.
// CF: the step (MODE_FULL or MODE_WORLD) that also reports its contacts (DESIGN.md section 7.15): one record of 10 rows per contact
// candidate k (plane candidates, then the candidates between multibodies), row r at 10 k + r, world coordinates: normal on b [3],
// point on b [3], distance, impulse on b [3] at the point on b.  The geometry rows are written where the candidate's distance is
// computed; every impulse row is zeroed there and the active contacts' rows are written after their group's PGS sweep or spring-damper
// loop.  Row r at pm.cf[r * ns + e] (value instances, fp32), or its dual part at io.jac[((n_q + n_qd + r) * m + j) * ns + e] behind the
// rows q' | qd' (JV instances).  Nothing else differs from the step.
// CEN: the centroidal quantities (DESIGN.md section 7.16), launched in MODE_NOCONTACT with qd in io.qd_in (null: zero).  Pass 1 adds
// every link's rigid inertia r_i about O (and the floating base's) into the body record and v_i x* (r_i v_i) into the velocity-only rate of
// momentum about O; pass 2 accumulates the composites Ic_i as MASS does, takes F = Ic_i S_i as column qd_idx of the momentum about O and
// adds Ic_i (v_i x S_i qd_i) to the rate.  A floating base's columns are the total inertia times the base twist's unit columns.  Then
// everything shifts to the centroid c: k_G = k_O - (c - O) x l.  Outputs pm.com [10], pm.A [6 n_qd] and pm.bias [6] (each may be null),
// row r at out[r * ns + e] (fp64 instances) or its dual part at out[(r * m + j) * ns + e] (JV instances).  ABA and integration are not
// compiled in.
// MOT: point velocities, accelerations and spatial point Jacobians (DESIGN.md section 7.17), launched in MODE_NOCONTACT with the point
// table as pm, qd in io.qd_in and qdd in io.tau_in (either null: zero; tangent input indices n_q + k and n_q + n_qd + k).  Pass 1 carries
// a_i = a_parent + S_i qdd_i + v_i x (S_i qd_i) as INV does but without gravity (a_base = 0, or the floating base's R_b qdd[0:6]); as it
// reaches link l it writes, for every point on l at x (relative to O), [w; x'] = [v.top; v.bot + w x x], [w'; x''] = [a.top; a.bot +
// a.top x x + w x x'] and the 6 x n_qd Jacobian (rows [w; x'], joint column [S.top; S.bot + S.top x x], floating-base columns [R_b | 0;
// -[x]x R_b | R_b] in the base-twist coordinates of qd[0:6]).  Outputs pm.J [6K n_qd], pm.vel [6K], pm.acc [6K] (each may be null), row r
// at out[r * ns + e] (fp64 instance) or its dual part at out[(r * m + j) * ns + e] (JV instance).  Returns before pass 2.
// EXT: the step with external wrenches (DESIGN.md section 7.18), point table and wrenches in pm.ext.  As pass 1 reaches link l it sums the
// wrenches about O of l's points at x (relative to O), [n + x x f; f] in RC, and stores the sum at RA precision in l's 6 RA words at arena
// word pm.ext.x_ext (a region behind the layout's x_total, present only in the EXT launches; links without points skip both the store
// and the load); pass 2 subtracts it from l's bias force pA
// (kinematics.hpp:132, pA = v x* I v - f_ext), and the floating base's points go into the base's bias force in the base frame.  Component r
// of point k's wrench is input direction n_in_ad + 6k + r (JV instances: entry 6k + r of the tangent pm.ext.t_W).  Nothing else differs
// from the step.
// REG (with INV): the joint-torque regressor Y(q, qd, qdd) and the energy regressors yT(q, qd), yV(q) of the inertial parameters
// (DESIGN.md section 7.19), launched as INV.  Column 10 b + c of body b (0: the floating base, i + 1: link i) is the unit barycentric
// parameter c of [m, m c, I about the body origin] in body axes, column 10 (n_links + 1) + 2 i (+ 1) link i's stiffness (damping).  Pass 1
// carries v_i and a_i as INV does; for each unit parameter it forms the rigid inertia r about O in world axes, f = r a_i + v_i x* (r v_i),
// and writes S_j . f for every row j (zero off the chain of i), R_b^T f in a floating base's rows, 1/2 v_i . (r v_i) and -g . (h + m O).
// Then the base's own columns (base frame) and the stiffness and damping columns.  Y [n_qd * n_pi] at io.jac, entry (r, c) at row
// r * n_pi + c, yT and yV [n_pi] at pm.yT and pm.yV (each may be null); row k at out[k * ns + e] (fp64 instance) or its dual part at
// out[(k * m + j) * ns + e] (JV instance).  Returns before pass 2.
// MINV (with MASS): the inverse mass matrix M^-1(q) (DESIGN.md section 7.20), launched as MASS.  After the floating-base block the lane
// factors the blocked lower triangle as the contact solve does (M = L L^T: off-diagonal blocks of L over M, inverted diagonal blocks in
// dinv), overwrites L's off-diagonal blocks with those of W = L^-1 column by column, and writes M^-1 = W^T W in place of the dense M: one
// sum per pair (r >= c) written to (r, c) and (c, r).  The padding dofs hold an identity, so the first n_qd rows and columns of the
// padded inverse are M^-1; they are not written.
// COR: the Coriolis matrix C(q, qd) of Echeandia & Wensing (DESIGN.md section 7.22), launched in MODE_NOCONTACT with qd in io.qd_in (null:
// zero).  Pass 1 as CEN's (v_i and the rigid inertias r_i about O in the link records).  Pass 2 carries, next to the composite Ic_i, the
// composite rate Ic_i' = sum r_k' (r' = v x* r - r v x, a rigid-inertia record with m' = 0) and momentum h_i = sum r_k v_k of the subtree
// in the accumulators' ABA words, so that the composite B_i u = 1/2 (Ic_i' u + u x* h_i).  With S' = v_i x S for the columns of link i and
// v_j x S for those of an ancestor j (the base twist's: v_b x S), C(a, a') = S_a . F_a' within link i and C(b, a) = S_b . F_a, C(a, b) =
// (B_i^T S_a - v_j x* (Ic_i S_a)) . S_b against its ancestors' columns b, F_a = Ic_i S_a' + B_i S_a (B_i^T = 1/2 (Ic_i' - h_i x*) is
// B_i with the skew part negated).  A floating base's own block after the sweep from the whole tree's composites.  Every entry is
// written: zeros first, C [n_qd * n_qd] at io.jac as MASS writes M (padding dofs not written).  ABA and integration are not compiled in.
// DER: the derivatives d tau / dq and d tau / dqd of INV's tau (DESIGN.md section 7.23), launched as INV, in the tangent coordinates of
// the velocities: the tangent of q along the motion with velocity e_k.  Pass 1 carries v_i and a_i as INV does and keeps a_i and f_i =
// r_i a_i + v_i x* (r_i v_i) per link in a region of 12 RC words per link at the end of the arena (x_total - 12 RCW n_links: the launch
// grows the layout, tds_der_layout_w).  Pass 2 carries COR's composites Ic_i, Ic_i' and h_i and the subtree force F_i = sum f_k.  A column
// S (link j's, or the base twist's) with the parent's velocity v_l and acceleration a_l (the base's: 0 and -g) moves the subtree of j
// rigidly (q) or adds S to its velocities (qd); what does not move with it is alpha = v_l x S, gamma = a_l x S + v_l x alpha (q) or S,
// psi = (v_l + v_j) x S (qd), and each body k of the subtree adds F(gamma, alpha) = r_k gamma + r_k' alpha + alpha x* (r_k v_k) to its
// force, the covariant S x* f_k besides (q).  So row b of link i against column S of an ancestor-or-self j is S_b . F_i(gamma, alpha)
// (qd: F_i(psi, S)), = (Ic_i S_b) . gamma + (Ic_i' S_b - S_b x* h_i) . alpha, and row b of a strict ancestor against S of link i is
// S_b . (F_i(gamma, alpha) + S x* F_i) (qd: S_b . F_i(psi, S)).  The stiffness and damping terms go into link i's own block, a spherical
// joint's axis-angle stiffness along its three tangents by a local dual number; a floating base's own block after the sweep from the
// whole tree's composites.  Every entry is written: zeros first, d tau / dq [n_qd * n_qd] at io.jac and d tau / dqd at io.g_in (either
// may be null), row-major as MASS writes M.  qdd is INV's fp32 tau_in, or the fp64 io.g_out [n_qd][ns] when that is not null (the
// forward dynamics' derivatives, section 7.24).  ABA and integration are not compiled in.
template <typename RA, typename RC, typename RS, typename RQ, bool SMEM, bool PAR = false, bool JV = false, bool MASS = false,
          bool KIN = false, bool INV = false, bool CF = false, bool CEN = false, bool MOT = false, bool EXT = false, bool REG = false,
          bool MINV = false, bool COR = false, bool DER = false>
__global__ void __launch_bounds__(128, 1)
tds_stepw_kernel(const __grid_constant__ DevModel M, const __grid_constant__ SimParams P,
                 const __grid_constant__ EnvParams E, const StepIO io, const int mode, const int use_pd,
                 char* __restrict__ gscratch, const __grid_constant__ typename ParArg<PAR, JV, KIN, CF, CEN, MOT, EXT, REG>::type pm = {}) {
  extern __shared__ __align__(16) char smem_raw[];
  const int lane = threadIdx.x & 31;
  const int warp_in_blk = threadIdx.x >> 5;
  const int env = blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = env < io.n;
  const int e = live ? env : io.n - 1;
  constexpr bool AD = is_dual<RQ>::value;
  constexpr bool TP = is_tape<RQ>::value;
  const int dir = AD ? (int)blockIdx.y + io.jac_dir0 : -1;     // differentiable instance: this lane's input direction
  Arena A;
  if (SMEM) { A.blk = smem_raw + (size_t)warp_in_blk * M.x_total * 32 * 4; A.stride = 32; A.col = lane; }
  else { A.blk = gscratch + ((size_t)blockIdx.y * ((size_t)gridDim.x * (blockDim.x >> 5)) + (size_t)(env >> 5)) * M.x_total * 32 * 4; A.stride = 32; A.col = lane; }  // per-warp block, same addressing as shared memory
  const int ST = A.stride;
  const int ns = io.n_stride;
  auto seed = [&](RQ x, int idx) -> RQ {   // d input_idx / d direction, or leaf idx of the tape, or the tangent's entry idx
    if constexpr (JV) return jv_seed(x, pm.jv.t_in, idx, pm.jv.m, dir, ns, e);
    else return ad_seed(x, idx, dir);
  };
  const int n_links = M.n_links;
  const int n = M.n_qd;
  const int nb = M.nb;
  const int n3 = 3 * nb;
  // VJP instance: input columns q | qd | tau or action (| kp, kd, max_force) are the first nodes of the lane's tape
  const int n_in_ad = M.n_q + n + (use_pd ? E.n_act + 3 : n - (M.floating ? 6 : 0));
  // (the instances without parameters keep their original statements: their code must not change)
  if constexpr (TP && PAR) tape_begin((TapeNode*)io.tape + ((size_t)(env >> 5) * io.tape_cap * 32 + lane), io.tape_cap, io.tape_overflow, n_in_ad + pm.n);
  else if constexpr (TP) tape_begin((TapeNode*)io.tape + ((size_t)(env >> 5) * io.tape_cap * 32 + lane), io.tape_cap, io.tape_overflow, n_in_ad);
  // reverse sweep from the cotangent of the outputs out_id(r), r < n_rows; the input adjoints are this lane's g_in column
  // (and its g_par column: the installed parameters are the leaves after the inputs)
  auto vjp_write = [&](int n_rows, auto out_id) {
    double* adj = io.tape_adj + ((size_t)(env >> 5) * io.tape_cap * 32 + lane);
    if constexpr (PAR) {
      const bool ok = tape_reverse(adj, n_rows, out_id, [&](int r) { return io.g_out[(size_t)r * ns + e]; }, n_in_ad + pm.n);
      if (ok && live && io.g_in)
        for (int k = 0; k < n_in_ad; ++k) io.g_in[(size_t)k * ns + e] = adj[(size_t)k * 32];
      if (ok && live && pm.grad)
        for (int k = 0; k < pm.n; ++k) pm.grad[(size_t)k * ns + e] = adj[(size_t)(n_in_ad + k) * 32];
    } else {
      const bool ok = tape_reverse(adj, n_rows, out_id, [&](int r) { return io.g_out[(size_t)r * ns + e]; }, n_in_ad);
      if (ok && live)
        for (int k = 0; k < n_in_ad; ++k) io.g_in[(size_t)k * ns + e] = adj[(size_t)k * 32];
    }
  };
  // Jacobian column of this lane's direction: parameter directions n_in_ad + s are column s of the parameter Jacobian (the JVP
  // instances: the tangent's column)
  const int jcol = (PAR && !JV && dir >= n_in_ad) ? dir - n_in_ad : dir;
  // physical quantities: the lane's installed value (the dual / taping instances seed it) or the model's.  RP keeps fp64 in the
  // plain instances, as the model stores these quantities.
  typedef typename std::conditional<AD || TP, RQ, double>::type RP;
  auto par_of = [&](int slot, double model_v) -> RP {
    if constexpr (PAR && JV) { if (slot >= 0) return jv_seed(RP(pm.values[(size_t)slot * ns + e]), pm.jv.t_par, slot, pm.jv.m, dir, ns, e); }
    else if constexpr (PAR) { if (slot >= 0) return ad_seed(RP(pm.values[(size_t)slot * ns + e]), n_in_ad + slot, dir); }
    return RP(model_v);
  };
  auto body_slot = [&](int b, int c) -> int {
    if constexpr (PAR) return pm.body[b][c];
    else return -1;
  };
  auto joint_slot = [&](int i, int c) -> int {
    if constexpr (PAR) return pm.joint[i][c];
    else return -1;
  };
  int par_friction = -1, par_restitution = -1;
  if constexpr (PAR) { par_friction = pm.friction; par_restitution = pm.restitution; }
  // joint stiffness (c = 0) / damping (c = 1) of link i, at fp32
  auto joint_par = [&](int i, int c, float model_v) -> RP {
    const int s = joint_slot(i, c);
    if (s >= 0) return f32_round(par_of(s, 0.0));
    return RP(model_v);
  };
  int phase_id = 0;
#define TDSW_PHASE() do { if (io.phase_clk && lane == 0) io.phase_clk[(size_t)(env >> 5) * 16 + (phase_id++)] = clock64(); } while (0)
  TDSW_PHASE();
  constexpr int RAW = (int)(sizeof(RA) / 4), RCW = (int)(sizeof(RC) / 4);
  RQ* const qv = A.ptr<RQ>(M.x_q);
  RQ* const qdv = A.ptr<RQ>(M.x_qd);
  RQ* const tauv = A.ptr<RQ>(M.x_tau);
  RC* const Sw = A.ptr<RC>(M.x_S);                 // S of link i at Sw + i*6*ST
  RC* const S3w = A.ptr<RC>(M.x_S3);               // spherical joints: three columns at S3w + s3_slot*18*ST
  // column c of link j's motion subspace (1 column, or 3 for a spherical joint)
  auto S_col = [&](int j, int c) -> Sv<RC> {
    return (M.flags[j] & TDS_LF_SPHERICAL) ? ld6<RC>(S3w + (M.s3_slot[j] * 3 + c) * 6 * ST, ST) : ld6<RC>(Sw + j * 6 * ST, ST);
  };
  auto n_cols = [&](int j) -> int { return (M.flags[j] & TDS_LF_FIXED) ? 0 : ((M.flags[j] & TDS_LF_SPHERICAL) ? 3 : 1); };
  const int LWD = M.x_link_words;
  const int VOFF = LWD - 6 * RAW;                  // word offset of v/c/a inside a link record
  // DER: a_i at derw + 12 i ST and f_i behind it (the region the DER launches add at the end of the layout)
  RC* const derw = [&]() -> RC* {
    if constexpr (DER) return A.ptr<RC>(M.x_total - 12 * RCW * n_links);
    else return nullptr;
  }();
  RS* const Mb = A.ptr<RS>(M.x_M);
  RS* const dinv = A.ptr<RS>(M.x_dinv);
  RS* const wv = A.ptr<RS>(M.x_w);
  // INV only (the step's own statements of these two stay inline: its code must not change).  quaternion_axis_angle(q) of spherical
  // joint i, the vector its stiffness multiplies (forward_dynamics.hpp:69-74, tiny_algebra.hpp:509-527)
  // (of the quaternion's components in any scalar type: DER evaluates it on a local dual number for its q-derivative)
  auto axis_angle_of = [&](auto qx, auto qy, auto qz, auto qw) {
    typedef decltype(qx) T;
    const T nrm = sqrt_t(qx * qx + qy * qy + qz * qz);
    const T theta = T(2) * atan2_t(nrm, qw);
    const T scaling = nrm < T(1.220703125e-4) ? T(1) / (T(0.5) + theta * theta * T(1.0 / 48.0)) : theta / nrm;   // eps^(1/4)
    return v3<T>(scaling * qx, scaling * qy, scaling * qz);
  };
  auto axis_angle = [&](int i) -> V3<RC> {
    const int q0 = M.q_idx[i];
    return axis_angle_of(RC(qv[q0 * ST]), RC(qv[(q0 + 1) * ST]), RC(qv[(q0 + 2) * ST]), RC(qv[(q0 + 3) * ST]));
  };
  // installed base quantities: (m, h, I about the origin) packed per lane as tds_rbi_pack does on the host (the block after pass 2)
  auto installed_base = [&](Rbi<RP>& bp) {
    RP b[10];
    for (int c = 0; c < 10; ++c) b[c] = par_of(body_slot(0, c), M.base_rbic[c]);
    const RP cc = b[1] * b[1] + b[2] * b[2] + b[3] * b[3];
    bp.m = b[0];
    bp.h = v3<RP>(b[0] * b[1], b[0] * b[2], b[0] * b[3]);
    bp.I.xx = b[4] + b[0] * (cc - b[1] * b[1]);
    bp.I.xy = b[5] - b[0] * b[1] * b[2];
    bp.I.xz = b[6] - b[0] * b[1] * b[3];
    bp.I.yy = b[7] + b[0] * (cc - b[2] * b[2]);
    bp.I.yz = b[8] - b[0] * b[2] * b[3];
    bp.I.zz = b[9] + b[0] * (cc - b[3] * b[3]);
  };

  // ---- load state, PD torques (locomotion_contact_simulation.h:168-258) ---------------------------
  // input directions of the differentiable instance: q | qd | tau or action | kp, kd, max_force (with PD)
  const int in0 = M.n_q + n;
  for (int k = 0; k < M.n_q; ++k) qv[k * ST] = seed(RQ(io.q_in[(size_t)k * ns + e]), k);
  for (int k = 0; k < n; ++k) qdv[k * ST] = (MASS || KIN) ? RQ(0.f) : seed(RQ(((INV || CEN || MOT || COR || DER) && !io.qd_in) ? 0.f : io.qd_in[(size_t)k * ns + e]), M.n_q + k);
  for (int k = 0; k < n; ++k) tauv[k * ST] = RQ(0.f);
  if (!MASS && use_pd) {
    const RQ kp = seed(RQ(E.kp), in0 + E.n_act), kd = seed(RQ(E.kd), in0 + E.n_act + 1), fmax_ = seed(RQ(E.max_force), in0 + E.n_act + 2);
    for (int k = 0; k < E.n_act; ++k) {
      const int li = E.act_link[k];
      RQ a = seed(RQ(io.tau_in[(size_t)k * ns + e]), in0 + k);
      a = max_t(min_t(a, RQ(E.action_limit)), RQ(-E.action_limit));
      const RQ q_des = RQ(E.initial_poses[k]) + a;
      RQ f = kp * (q_des - qv[M.q_idx[li] * ST]) + kd * (RQ(0.f) - qdv[M.qd_idx[li] * ST]);
      f = min_t(max_t(f, -fmax_), fmax_);
      tauv[M.qd_idx[li] * ST] = f;
    }
  } else if (!MASS && !INV && !MOT && !DER && io.tau_in) {
    const int off = M.floating ? 6 : 0;
    for (int k = off; k < n; ++k) tauv[k * ST] = seed(RQ(io.tau_in[(size_t)(k - off) * ns + e]), in0 + k - off);
  }
  if constexpr (!KIN && !INV && !MOT) {   // (the KIN, INV and MOT lanes return before pass 2 reads the accumulators)
    for (int s = 0; s < M.n_acc; ++s) {
      RA* pa = A.ptr<RA>(M.x_acc + s * M.x_acc_words);
      for (int k = 0; k < 27; ++k) pa[k * ST] = RA(0);
      RC* pc = A.ptr<RC>(M.x_acc + s * M.x_acc_words + M.x_acc_ic_word);
      for (int k = 0; k < 10; ++k) pc[k * ST] = RC(0);
    }
  }
  const bool world_step = mode == MODE_WORLD;   // World::step(dt) on its own (src/world.hpp:302-363): q, qd in -> qd out
  const bool want_contacts = (mode == MODE_FULL || world_step) && (M.has_plane || M.n_pair_points > 0);
  TDSW_PHASE();  // 1

  // ---- common-frame origin O (world coordinates) -----------------------------------------------------
  M3<RC> Rb = m3_identity<RC>();
  V3<RC> O = v3<RC>(RC(0), RC(0), RC(0));
  if (M.floating) {
    Rb = quat_to_matrix<RC>(RC(qv[0]), RC(qv[ST]), RC(qv[2 * ST]), RC(qv[3 * ST]));
    O = v3<RC>(RC(qv[4 * ST]), RC(qv[5 * ST]), RC(qv[6 * ST]));
  } else {
    // end of the translation-only root chain: constant rotations, no trigonometry
    M3<RC> Rc = m3_identity<RC>();
    const int kp = M.n_prefix < n_links ? M.n_prefix + 1 : n_links;
    for (int i = 0; i < kp; ++i) {
      const double* xt = M.XT[i];
      O = O + mul(Rc, v3<RC>(RC(xt[9]), RC(xt[10]), RC(xt[11])));
      if (i == M.n_prefix) break;
      if (!(M.flags[i] & TDS_LF_XT_IDENT)) {
        M3<RC> r; r.xx = RC(xt[0]); r.xy = RC(xt[1]); r.xz = RC(xt[2]); r.yx = RC(xt[3]); r.yy = RC(xt[4]); r.yz = RC(xt[5]); r.zx = RC(xt[6]); r.zy = RC(xt[7]); r.zz = RC(xt[8]);
        Rc = mul(Rc, r);
      }
      if (M.flags[i] & TDS_LF_PRISMATIC) {
        const RC qi = RC(qv[M.q_idx[i] * ST]);
        O = O + mul(Rc, v3<RC>(RC(M.axis[i][0]) * qi, RC(M.axis[i][1]) * qi, RC(M.axis[i][2]) * qi));
      }
    }
  }

  // ---- pass 1: root -> leaf.  kinematics.hpp:18-148 in the common frame + contact detection ------------
  const V3<RC> pn = v3<RC>(RC(M.plane_n[0]), RC(M.plane_n[1]), RC(M.plane_n[2]));
  const RC plane_off = dot(O, pn) - RC(M.plane_c);   // n.(O + x) - c = n.x + plane_off
  int n_active = 0, pt_index = 0;
  // CF: row r of the records; the geometry of candidate k (xb relative to O) with zero impulse rows; the active candidates as bits
  // (plane candidate k, candidate pt between multibodies), from which the impulse rows recover each compacted contact's candidate
  auto cf_put = [&](int r, auto x) {
    if constexpr (CF) {
      if (!live) return;
      if constexpr (AD) io.jac[((size_t)(M.n_q + n + r) * io.jac_n_in + jcol) * ns + e] = x.TDS_CF_DUAL_PART;
      else pm.cf[(size_t)r * ns + e] = (float)val_of(x);
    }
  };
  auto cf_geom = [&](int k, const V3<RC>& n_b, const V3<RC>& xb, const RC& dist) {
    if constexpr (CF) {
      cf_put(10 * k, n_b.x); cf_put(10 * k + 1, n_b.y); cf_put(10 * k + 2, n_b.z);
      cf_put(10 * k + 3, xb.x + O.x); cf_put(10 * k + 4, xb.y + O.y); cf_put(10 * k + 5, xb.z + O.z);
      cf_put(10 * k + 6, dist);
      for (int r = 7; r < 10; ++r) cf_put(10 * k + r, RC(0));
    }
  };
  unsigned long long cf_plane = 0ull, cf_pair = 0ull;
  auto emit_point = [&](int li, const V3<RC>& pos, const RC rad) {
    if (!M.has_plane) return;
    const RC dist = dot(pos, pn) + plane_off - rad;       // contact_plane_sphere, contact_point.hpp:112-116
    if (io.contact_dist && live) io.contact_dist[(size_t)pt_index * ns + e] = (float)val_of(dist);
    if constexpr (CF) {
      cf_geom(pt_index, v3<RC>(-pn.x, -pn.y, -pn.z), pos - pn * rad, dist);
      if (dist < RC(0) && n_active < M.max_contacts) cf_plane |= 1ull << pt_index;
    }
    ++pt_index;
    if (dist < RC(0) && n_active < M.max_contacts) {
      RC* pc = A.ptr<RC>(M.x_con + n_active * 5 * RCW);
      st3<RC>(pc, ST, pos - pn * rad);                     // world_point_on_b, relative to O
      pc[3 * ST] = dist;
      pc[4 * ST] = RC(li);
      ++n_active;
    }
  };
  auto emit_geoms = [&](int li, const M3<RC>& R, const V3<RC>& pr) {
    for (int g = M.geom_begin[li + 1]; g < M.geom_begin[li + 2]; ++g) {
      const int ty = M.g_type[g];
      if (ty != TDSG_SPHERE && ty != TDSG_CAPSULE && ty != TDSG_BOX) continue;
      const V3<RC> c = pr + mul(R, v3<RC>(RC(M.g_t[g][0]), RC(M.g_t[g][1]), RC(M.g_t[g][2])));
      const RC rad = RC(M.g_radius[g]);
      if (M.g_wslot[g] >= 0) {         // kept for the contacts between multibodies (after this pass)
        RC* pw = A.ptr<RC>(M.x_gw + M.g_wslot[g] * 12 * RCW);
        st3<RC>(pw, ST, c);
        if (ty == TDSG_CAPSULE) st3<RC>(pw + 3 * ST, ST, mul(R, v3<RC>(RC(M.g_half[g][0]), RC(M.g_half[g][1]), RC(M.g_half[g][2]))));
        if (ty == TDSG_BOX) {
          const double* b = M.g_box[g];
          st3<RC>(pw + 3 * ST, ST, mul(R, v3<RC>(RC(b[0]), RC(b[1]), RC(b[2]))));
          st3<RC>(pw + 6 * ST, ST, mul(R, v3<RC>(RC(b[3]), RC(b[4]), RC(b[5]))));
          st3<RC>(pw + 9 * ST, ST, mul(R, v3<RC>(RC(b[6]), RC(b[7]), RC(b[8]))));
        }
      }
      if (ty == TDSG_SPHERE) emit_point(li, c, rad);
      else if (ty == TDSG_CAPSULE) {   // contact_plane_capsule, contact_point.hpp:128-161: end spheres at +L/2, then -L/2
        const V3<RC> half = mul(R, v3<RC>(RC(M.g_half[g][0]), RC(M.g_half[g][1]), RC(M.g_half[g][2])));
        emit_point(li, c + half, rad);
        emit_point(li, c - half, rad);
      } else {                         // contact_plane_box, contact_point.hpp:164-198: corner spheres, x outermost, z innermost
        const double* b = M.g_box[g];
        const V3<RC> ex = mul(R, v3<RC>(RC(b[0]), RC(b[1]), RC(b[2])));
        const V3<RC> ey = mul(R, v3<RC>(RC(b[3]), RC(b[4]), RC(b[5])));
        const V3<RC> ez = mul(R, v3<RC>(RC(b[6]), RC(b[7]), RC(b[8])));
        for (int k = 0; k < 8; ++k) {
          V3<RC> pos = (k & 4) ? c - ex : c + ex;
          pos = (k & 2) ? pos - ey : pos + ey;
          pos = (k & 1) ? pos - ez : pos + ez;
          emit_point(li, pos, rad);
        }
      }
    }
  };
  // KIN: the outputs of link l (-1: the base) at its world rotation R and position p (relative to O).  The Jacobian of a point on l
  // reads the stored S of l and of its ancestors, all written by the time pass 1 reaches l (links are ordered parent first), so it is
  // written here too and the points' positions need no storage.
  auto kin_link = [&](int l, const M3<RC>& R, const V3<RC>& p) {
    if constexpr (KIN) {
      if (!live) return;
      auto put = [&](double* o, size_t r, const RC& x) {
        if constexpr (AD) o[(r * io.jac_n_in + jcol) * ns + e] = x.d;
        else o[r * ns + e] = x;
      };
      if (pm.xf && l >= 0) {   // the layout of io.link_xf: R row-major, then the position
        const size_t r0 = (size_t)l * 12;
        put(pm.xf, r0, R.xx); put(pm.xf, r0 + 1, R.xy); put(pm.xf, r0 + 2, R.xz);
        put(pm.xf, r0 + 3, R.yx); put(pm.xf, r0 + 4, R.yy); put(pm.xf, r0 + 5, R.yz);
        put(pm.xf, r0 + 6, R.zx); put(pm.xf, r0 + 7, R.zy); put(pm.xf, r0 + 8, R.zz);
        put(pm.xf, r0 + 9, p.x + O.x); put(pm.xf, r0 + 10, p.y + O.y); put(pm.xf, r0 + 11, p.z + O.z);
      }
      for (int k = 0; k < pm.K; ++k) {
        if (pm.link[k] != l) continue;
        const V3<RC> xr = p + mul(R, v3<RC>(RC(pm.local[3 * k]), RC(pm.local[3 * k + 1]), RC(pm.local[3 * k + 2])));
        if (pm.x) { put(pm.x, 3 * k, xr.x + O.x); put(pm.x, 3 * k + 1, xr.y + O.y); put(pm.x, 3 * k + 2, xr.z + O.z); }
        if (!pm.J) continue;
        // rows 3k .. 3k + 2 of n_qd columns: zero outside the point's chain (and outside its multibody)
        const size_t r0 = (size_t)3 * k * n;
        auto put_col = [&](int c, const V3<RC>& col) { put(pm.J, r0 + c, col.x); put(pm.J, r0 + n + c, col.y); put(pm.J, r0 + 2 * n + c, col.z); };
        const V3<RC> z = v3<RC>(RC(0), RC(0), RC(0));
        for (int c = 0; c < n; ++c) put_col(c, z);
        if (M.floating) {   // jacobian.hpp:39-58: [-[x - r0]x^T | I3] with the base rotation ignored (O is the base origin r0)
          put_col(0, v3<RC>(RC(0), -xr.z, xr.y)); put_col(1, v3<RC>(xr.z, RC(0), -xr.x)); put_col(2, v3<RC>(-xr.y, xr.x, RC(0)));
          put_col(3, v3<RC>(RC(1), RC(0), RC(0))); put_col(4, v3<RC>(RC(0), RC(1), RC(0))); put_col(5, v3<RC>(RC(0), RC(0), RC(1)));
        }
        for (int j = l; j >= 0; j = M.parent[j]) {   // jacobian.hpp:63-80: column = S_j evaluated at the point (fixed links: none)
          for (int cj = 0; cj < n_cols(j); ++cj) {
            const Sv<RC> S = S_col(j, cj);
            put_col(M.qd_idx[j] + cj, S.bot + cross(S.top, xr));
          }
        }
      }
    }
  };
  // MOT: the outputs of the points on link l (-1: the base) at its world rotation R, position p (relative to O), spatial velocity v and
  // acceleration a (common frame).  The Jacobian reads the stored S of l and its ancestors, as kin_link does.
  auto mot_link = [&](int l, const M3<RC>& R, const V3<RC>& p, const Sv<RC>& v, const Sv<RC>& a) {
    if constexpr (MOT) {
      if (!live) return;
      auto put = [&](double* o, size_t r, const RC& x) {
        if constexpr (AD) o[(r * io.jac_n_in + jcol) * ns + e] = x.d;
        else o[r * ns + e] = x;
      };
      auto put6 = [&](double* o, size_t r0, size_t stride, const V3<RC>& top, const V3<RC>& bot) {
        put(o, r0, top.x); put(o, r0 + stride, top.y); put(o, r0 + 2 * stride, top.z);
        put(o, r0 + 3 * stride, bot.x); put(o, r0 + 4 * stride, bot.y); put(o, r0 + 5 * stride, bot.z);
      };
      for (int k = 0; k < pm.K; ++k) {
        if (pm.link[k] != l) continue;
        const V3<RC> xr = p + mul(R, v3<RC>(RC(pm.local[3 * k]), RC(pm.local[3 * k + 1]), RC(pm.local[3 * k + 2])));
        const V3<RC> xd = v.bot + cross(v.top, xr);
        if (pm.vel) put6(pm.vel, 6 * k, 1, v.top, xd);
        if (pm.acc) put6(pm.acc, 6 * k, 1, a.top, a.bot + cross(a.top, xr) + cross(v.top, xd));
        if (!pm.J) continue;
        // rows 6k .. 6k + 5 of n_qd columns: zero outside the point's chain (and outside its multibody)
        const size_t r0 = (size_t)6 * k * n;
        const V3<RC> z = v3<RC>(RC(0), RC(0), RC(0));
        for (int c = 0; c < n; ++c) put6(pm.J, r0 + c, n, z, z);
        if (M.floating) {   // the base twist's unit columns [R_b e_c; 0] and [0; R_b e_c], moved to the point
          for (int c = 0; c < 3; ++c) {
            const V3<RC> u = c == 0 ? col_x(Rb) : (c == 1 ? col_y(Rb) : col_z(Rb));
            put6(pm.J, r0 + c, n, u, cross(u, xr));
            put6(pm.J, r0 + 3 + c, n, z, u);
          }
        }
        for (int j = l; j >= 0; j = M.parent[j]) {   // column = S_j at the point (fixed links: none)
          for (int cj = 0; cj < n_cols(j); ++cj) {
            const Sv<RC> S = S_col(j, cj);
            put6(pm.J, r0 + M.qd_idx[j] + cj, n, S.top, S.bot + cross(S.top, xr));
          }
        }
      }
    }
  };
  // EXT: the wrench about O of point k on a body at world rotation R and position p (relative to O), [n + x x f; f] at x = p + R local
  // (JV: seeded with the tangent's entries 6k + r), and their sum over the points on body l (-1: the base)
  auto ext_wrench = [&](int k, const M3<RC>& R, const V3<RC>& p) -> Sv<RC> {
    Sv<RC> w;
    if constexpr (EXT) {
      RC c[6];
      for (int r = 0; r < 6; ++r) {
        const RQ x = RQ(pm.ext.W[(size_t)(6 * k + r) * ns + e]);
        if constexpr (JV) c[r] = RC(jv_seed(x, pm.ext.t_W, 6 * k + r, pm.jv.m, dir, ns, e));
        else c[r] = RC(x);
      }
      const V3<RC> x = p + mul(R, v3<RC>(RC(pm.ext.local[3 * k]), RC(pm.ext.local[3 * k + 1]), RC(pm.ext.local[3 * k + 2])));
      const V3<RC> f = v3<RC>(c[3], c[4], c[5]);
      w.top = v3<RC>(c[0], c[1], c[2]) + cross(x, f);
      w.bot = f;
    }
    return w;
  };
  auto ext_sum = [&](int l, const M3<RC>& R, const V3<RC>& p) -> Sv<RC> {
    Sv<RC> w;
    w.top = v3<RC>(RC(0), RC(0), RC(0)); w.bot = w.top;
    if constexpr (EXT)
      for (int k = 0; k < pm.ext.K; ++k)
        if (pm.ext.link[k] == l) w = w + ext_wrench(k, R, p);
    return w;
  };
  // REG: the number of parameter columns; row k of an output; the rigid inertia about O in world axes of unit parameter c of a body at
  // world rotation R and position p (relative to O): the linear map of the rigid-inertia statements of pass 1 applied to a unit
  // [m, m c, I about the body origin]
  const int n_pi = 12 * n_links + 10;
  auto reg_put = [&](double* o, size_t k, const RC& x) {
    if constexpr (REG) {
      if (!o || !live) return;
      if constexpr (AD) o[(k * io.jac_n_in + jcol) * ns + e] = x.d;
      else o[k * ns + e] = x;
    }
  };
  auto reg_unit = [&](int c, const M3<RC>& R, const V3<RC>& p) -> Rbi<RC> {
    Rbi<RC> r;
    const V3<RC> z = v3<RC>(RC(0), RC(0), RC(0));
    // I = s (u w^T + w u^T) + d 1
    V3<RC> u = z, w = z;
    RC s = RC(0), d = RC(0);
    r.m = RC(0); r.h = z;
    if (c == 0) { r.m = RC(1); r.h = p; u = p; w = p; s = RC(-0.5); d = dot(p, p); }   // m (|p|^2 1 - p p^T)
    else if (c < 4) {                                                                    // 2 (p . h) 1 - p h^T - h p^T
      r.h = c == 1 ? col_x(R) : (c == 2 ? col_y(R) : col_z(R));
      u = p; w = r.h; s = RC(-1); d = RC(2) * dot(p, r.h);
    } else {                                                                             // R E R^T, E the unit symmetric entry
      const int a = c < 7 ? 0 : (c < 9 ? 1 : 2), b = c < 7 ? c - 4 : (c < 9 ? c - 6 : 2);
      u = a == 0 ? col_x(R) : (a == 1 ? col_y(R) : col_z(R));
      w = b == 0 ? col_x(R) : (b == 1 ? col_y(R) : col_z(R));
      s = a == b ? RC(0.5) : RC(1);
    }
    r.I.xx = s * (u.x * w.x + w.x * u.x) + d; r.I.yy = s * (u.y * w.y + w.y * u.y) + d; r.I.zz = s * (u.z * w.z + w.z * u.z) + d;
    r.I.xy = s * (u.x * w.y + w.x * u.y); r.I.xz = s * (u.x * w.z + w.x * u.z); r.I.yz = s * (u.y * w.z + w.y * u.z);
    return r;
  };
  // REG: the ten columns of body b (0: the base, i + 1: link i) with velocity v and acceleration a, at rotation R and position p: the
  // joint rows of link i's chain (l = i; l = -1: none) and of a floating base (S_j . f, R_b^T f), zeros elsewhere, and the energy rows
  auto reg_body = [&](int b, int l, const M3<RC>& R, const V3<RC>& p, const Sv<RC>& v, const Sv<RC>& a, bool base_frame) {
    if constexpr (REG) {
      const V3<RC> g = v3<RC>(RC(P.gravity[0]), RC(P.gravity[1]), RC(P.gravity[2]));
      for (int c = 0; c < 10; ++c) {
        const int col = 10 * b + c;
        const Rbi<RC> r = reg_unit(c, R, p);
        const Sv<RC> rv = rbi_mul(r, v);
        const Sv<RC> f = rbi_mul(r, a) + cross_mf(v, rv);
        if (M.floating) {
          const V3<RC> ft = base_frame ? f.top : mulT(Rb, f.top), fb = base_frame ? f.bot : mulT(Rb, f.bot);
          const RC fr[6] = {ft.x, ft.y, ft.z, fb.x, fb.y, fb.z};
          for (int k = 0; k < 6; ++k) reg_put(io.jac, (size_t)k * n_pi + col, fr[k]);
        }
        int anc = l;
        for (int j = n_links - 1; j >= 0; --j) {   // links are ordered parent first: the chain of l, walked downwards
          const bool on = j == anc;
          if (on) anc = M.parent[j];
          for (int cj = 0; cj < n_cols(j); ++cj)
            reg_put(io.jac, (size_t)(M.qd_idx[j] + cj) * n_pi + col, on ? dot(S_col(j, cj), f) : RC(0));
        }
        reg_put(pm.yT, col, RC(0.5) * dot(v, rv));
        const V3<RC> hw = base_frame ? mul(Rb, r.h) : r.h;
        reg_put(pm.yV, col, -dot(g, hw + O * r.m));
      }
    }
  };
  M3<RC> R_prev = Rb;
  V3<RC> p_prev = M.floating ? v3<RC>(RC(0), RC(0), RC(0)) : v3<RC>(-O.x, -O.y, -O.z);
  Sv<RA> v_prev;
  if (M.floating) {  // base-frame spatial velocity qd[0:6] (kinematics.hpp:45-47) expressed in the common frame
    const M3<RA> RbA = cvt<RA>(Rb);
    v_prev.top = mul(RbA, v3<RA>(RA(qdv[0]), RA(qdv[ST]), RA(qdv[2 * ST])));
    v_prev.bot = mul(RbA, v3<RA>(RA(qdv[3 * ST]), RA(qdv[4 * ST]), RA(qdv[5 * ST])));
  } else {
    v_prev.top = v3<RA>(RA(0), RA(0), RA(0)); v_prev.bot = v_prev.top;
  }
  const M3<RC> R_base = R_prev;
  const V3<RC> p_base = p_prev;
  const Sv<RA> v_base = v_prev;
  { RC* px = A.ptr<RC>(M.x_xw); st9<RC>(px, ST, R_base); st3<RC>(px + 9 * ST, ST, p_base); }
  if (want_contacts) emit_geoms(-1, R_base, p_base);
  if constexpr (KIN) kin_link(-1, R_base, p_base);
  // INV: qdd of dof k (seeded at input n_q + n_qd + k); the acceleration of the previous link, of the base; the sum of the link forces.
  // DER reads qdd in fp64 from io.g_out [n_qd][ns] when the launch gives it (the forward dynamics' derivatives, DESIGN.md section 7.24;
  // no DER lane reads g_out otherwise), else from tau_in as INV does.
  auto qdd_in = [&](int k) -> RQ {
    if constexpr (DER) { if (io.g_out) return seed(RQ(io.g_out[(size_t)k * ns + e]), M.n_q + n + k); }
    return seed(RQ(io.tau_in ? io.tau_in[(size_t)k * ns + e] : 0.f), M.n_q + n + k);
  };
  // (empty placeholders in the other instances, whose code must not change)
  typedef typename std::conditional<INV || MOT || DER, Sv<RC>, NoPar>::type SvInv;
  const SvInv a_base_inv = [&]() -> SvInv {
    if constexpr (MOT) {   // the base's acceleration without gravity: zero, or the base-frame qdd[0:6] in the common frame
      static_assert(std::is_same<RA, RC>::value && std::is_same<RC, RQ>::value, "the MOT instances run in one scalar type");
      Sv<RC> a;
      a.top = v3<RC>(RC(0), RC(0), RC(0));
      a.bot = a.top;
      if (M.floating) {
        a.top = mul(Rb, v3<RC>(qdd_in(0), qdd_in(1), qdd_in(2)));
        a.bot = mul(Rb, v3<RC>(qdd_in(3), qdd_in(4), qdd_in(5)));
      }
      return a;
    } else if constexpr (INV || DER) {
      static_assert(std::is_same<RA, RC>::value && std::is_same<RC, RQ>::value, "the INV and DER instances run in one scalar type");
      const V3<RC> g = v3<RC>(RC(P.gravity[0]), RC(P.gravity[1]), RC(P.gravity[2]));
      Sv<RC> a;
      a.top = v3<RC>(RC(0), RC(0), RC(0));
      a.bot = v3<RC>(-g.x, -g.y, -g.z);
      if (M.floating) {   // the base-frame spatial acceleration qdd[0:6] in the common frame (O is the base origin)
        a.top = mul(Rb, v3<RC>(qdd_in(0), qdd_in(1), qdd_in(2)));
        a.bot = mul(Rb, v3<RC>(qdd_in(3), qdd_in(4), qdd_in(5))) - g;
      }
      return a;
    } else {
      return SvInv{};
    }
  }();
  SvInv a_prev_inv = a_base_inv, f_links = SvInv{};
  if constexpr (INV) { f_links.top = v3<RC>(RC(0), RC(0), RC(0)); f_links.bot = f_links.top; }
  if constexpr (MOT) mot_link(-1, R_base, p_base, v_base, a_base_inv);
  // CEN: the rigid inertia of the counted bodies about O in world axes (the root composite) and the velocity-only rate of momentum about O
  typename std::conditional<CEN, Rbi<RC>, NoPar>::type cen_I{};
  typename std::conditional<CEN, Sv<RC>, NoPar>::type cen_f{};
  if constexpr (CEN) {
    static_assert(std::is_same<RA, RC>::value && std::is_same<RC, RQ>::value, "the CEN instances run in one scalar type");
    cen_I.m = RC(0); cen_I.h = v3<RC>(RC(0), RC(0), RC(0)); cen_I.I = {RC(0), RC(0), RC(0), RC(0), RC(0), RC(0)};
    cen_f.top = cen_I.h; cen_f.bot = cen_I.h;
    if (M.floating) {   // the base: its inertia about its origin O rotated to world axes, and its term v_b x* (I_b v_b) (qdd = 0)
      Rbi<RC> Ib = model_rbi_of<RC>(M.base_rbi);
      if constexpr (PAR) { if (pm.any_base) installed_base(Ib); }
      cen_I.m = Ib.m; cen_I.h = mul(Rb, Ib.h); cen_I.I = rot_sym(Rb, Ib.I);
      cen_f = cross_mf(v_base, rbi_mul(cen_I, v_base));
    }
  }
  for (int i = 0; i < n_links; ++i) {
    const int p = M.parent[i];
    const int fl = M.flags[i];
    M3<RC> Rp; V3<RC> pp; Sv<RA> vp;
    if (fl & TDS_LF_PARENT_ADJ) { Rp = R_prev; pp = p_prev; vp = v_prev; }
    else if (p >= 0) {
      const RC* px = A.ptr<RC>(M.x_xw + (M.xw_slot[p] + 1) * 12 * RCW);
      Rp = ld9<RC>(px, ST); pp = ld3<RC>(px + 9 * ST, ST);
      vp = ld6<RA>(A.ptr<RA>(M.x_link + p * LWD + VOFF), ST);
    } else { Rp = R_base; pp = p_base; vp = v_base; }
    const double* xt = M.XT[i];
    V3<RC> pi = pp + mul(Rp, v3<RC>(RC(xt[9]), RC(xt[10]), RC(xt[11])));
    M3<RC> Ri = Rp;
    if (!(fl & TDS_LF_XT_IDENT)) {
      M3<RC> r; r.xx = RC(xt[0]); r.xy = RC(xt[1]); r.xz = RC(xt[2]); r.yx = RC(xt[3]); r.yy = RC(xt[4]); r.yz = RC(xt[5]); r.zx = RC(xt[6]); r.zy = RC(xt[7]); r.zz = RC(xt[8]);
      Ri = mul(Rp, r);
    }
    Sv<RC> S; S.top = v3<RC>(RC(0), RC(0), RC(0)); S.bot = S.top;
    if (!(fl & TDS_LF_FIXED)) {   // Link::jcalc, link.hpp:229-336
      const RC qi = RC(qv[M.q_idx[i] * ST]);
      const int jt = M.jtype[i];
      const V3<RC> ax = v3<RC>(RC(M.axis[i][0]), RC(M.axis[i][1]), RC(M.axis[i][2]));
      if (fl & TDS_LF_SPHERICAL) {   // X_J = quat_to_matrix(q[0..3]) (link.hpp:268-272); S = [1 0]^T in the link frame
        const int q0 = M.q_idx[i];
        Ri = mul(Ri, quat_to_matrix<RC>(RC(qv[q0 * ST]), RC(qv[(q0 + 1) * ST]), RC(qv[(q0 + 2) * ST]), RC(qv[(q0 + 3) * ST])));
        RC* const s3 = S3w + M.s3_slot[i] * 18 * ST;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
          const V3<RC> w = a == 0 ? col_x(Ri) : (a == 1 ? col_y(Ri) : col_z(Ri));
          Sv<RC> Sa; Sa.top = w; Sa.bot = cross(pi, w);
          st6<RC>(s3 + a * 6 * ST, ST, Sa);
        }
      } else if (fl & TDS_LF_PRISMATIC) {
        const V3<RC> d = mul(Ri, ax);
        pi = axpy(d, qi, pi);
        S.bot = d;
      } else {
        const V3<RC> w = mul(Ri, ax);          // the joint axis is invariant under X_J
        if (jt == TDSJ_REVOLUTE_AXIS) {        // TinyQuaternion::setRotation(axis, angle), tiny_quaternion.h:178-183
          const RC dl = sqrt_t(dot(ax, ax));
          RC s, c;
          sincos_t(qi * RC(0.5), &s, &c);
          s = s / dl;
          Ri = mul(Ri, quat_to_matrix<RC>(ax.x * s, ax.y * s, ax.z * s, c));
        } else {
          RC s, c;
          sincos_t(qi, &s, &c);
          const V3<RC> cx = col_x(Ri), cy = col_y(Ri), cz = col_z(Ri);
          if (jt == TDSJ_REVOLUTE_X) set_cols(Ri, cx, axpy(cz, s, cy * c), axpy(cy, -s, cz * c));          // y' = c y + s z, z' = -s y + c z
          else if (jt == TDSJ_REVOLUTE_Y) set_cols(Ri, axpy(cz, -s, cx * c), cy, axpy(cx, s, cz * c));     // x' = c x - s z, z' = s x + c z
          else set_cols(Ri, axpy(cy, s, cx * c), axpy(cx, -s, cy * c), cz);                                 // x' = c x + s y, y' = -s x + c y
        }
        S.top = w;
        S.bot = cross(pi, w);
      }
    }
    st6<RC>(Sw + i * 6 * ST, ST, S);
    if (M.xw_slot[i] >= 0) { RC* px = A.ptr<RC>(M.x_xw + (M.xw_slot[i] + 1) * 12 * RCW); st9<RC>(px, ST, Ri); st3<RC>(px + 9 * ST, ST, pi); }
    // rigid-body inertia about O in world axes: com c = p_i + R_i com_l, I = R Icom R^T + m (|c|^2 1 - c c^T)
    typename std::conditional<INV, Rbi<RC>, NoPar>::type r_inv;   // (INV: kept for f_i below)
    if constexpr (!KIN && !MOT) {
      const double* rb = M.rbic[i];
      auto rbc = [&](int c) -> RP { return par_of(body_slot(i + 1, c), rb[c]); };
      Rbi<RC> r;
      r.m = RC(rbc(0));
      const V3<RC> c = pi + mul(Ri, v3<RC>(RC(rbc(1)), RC(rbc(2)), RC(rbc(3))));
      r.h = c * r.m;
      // R Icom R^T enters every product additively (no cancellation) -> RA precision is enough; the parallel-axis
      // terms m(|c|^2 1 - c c^T) and h = m c cancel against each other in M_ij and stay in RC.
      S3<RA> Icf; Icf.xx = RA(rbc(4)); Icf.xy = RA(rbc(5)); Icf.xz = RA(rbc(6)); Icf.yy = RA(rbc(7)); Icf.yz = RA(rbc(8)); Icf.zz = RA(rbc(9));
      const S3<RA> Irot = rot_sym(cvt<RA>(Ri), Icf);
      r.I.xx = RC(Irot.xx); r.I.xy = RC(Irot.xy); r.I.xz = RC(Irot.xz); r.I.yy = RC(Irot.yy); r.I.yz = RC(Irot.yz); r.I.zz = RC(Irot.zz);
      const RC cc = dot(c, c);
      r.I.xx += r.m * (cc - c.x * c.x); r.I.yy += r.m * (cc - c.y * c.y); r.I.zz += r.m * (cc - c.z * c.z);
      r.I.xy -= r.m * c.x * c.y; r.I.xz -= r.m * c.x * c.z; r.I.yz -= r.m * c.y * c.z;
      if constexpr (INV) r_inv = r;
      else st_rbi<RC>(A.ptr<RC>(M.x_link + i * LWD), ST, r);
    }
    Sv<RA> v = vp;
    if (fl & TDS_LF_SPHERICAL) {
      for (int a = 0; a < 3; ++a) {
        const RA qda = RA(qdv[(M.qd_idx[i] + a) * ST]);
        const Sv<RA> Sf = cvt_sv<RA>(S_col(i, a));
        v.top = axpy(Sf.top, qda, v.top);
        v.bot = axpy(Sf.bot, qda, v.bot);
      }
    } else if (!(fl & TDS_LF_FIXED)) {
      const RA qdi = RA(qdv[M.qd_idx[i] * ST]);
      const Sv<RA> Sf = cvt_sv<RA>(S);
      v.top = axpy(Sf.top, qdi, v.top);
      v.bot = axpy(Sf.bot, qdi, v.bot);
    }
    st6<RA>(A.ptr<RA>(M.x_link + i * LWD + VOFF), ST, v);
    if constexpr (EXT) {
      if ((pm.ext.links_with_points >> i) & 1ull) st6<RA>(A.ptr<RA>(pm.ext.x_ext + i * 6 * RAW), ST, cvt_sv<RA>(ext_sum(i, Ri, pi)));
    }
    if constexpr (CEN) {   // the link's share of the body record and its term v_i x* (r_i v_i) of the rate
      const Rbi<RC> r = ld_rbi<RC>(A.ptr<RC>(M.x_link + i * LWD), ST);
      rbi_add(cen_I, r);
      cen_f = cen_f + cross_mf(v, rbi_mul(r, v));
    }
    if (want_contacts) emit_geoms(i, Ri, pi);
    if (io.link_xf && live) {
      float* o = io.link_xf + (size_t)i * 12 * ns + e;
      o[0] = (float)val_of(Ri.xx); o[(size_t)1 * ns] = (float)val_of(Ri.xy); o[(size_t)2 * ns] = (float)val_of(Ri.xz);
      o[(size_t)3 * ns] = (float)val_of(Ri.yx); o[(size_t)4 * ns] = (float)val_of(Ri.yy); o[(size_t)5 * ns] = (float)val_of(Ri.yz);
      o[(size_t)6 * ns] = (float)val_of(Ri.zx); o[(size_t)7 * ns] = (float)val_of(Ri.zy); o[(size_t)8 * ns] = (float)val_of(Ri.zz);
      o[(size_t)9 * ns] = (float)val_of(pi.x + O.x); o[(size_t)10 * ns] = (float)val_of(pi.y + O.y); o[(size_t)11 * ns] = (float)val_of(pi.z + O.z);
    }
    if constexpr (KIN) kin_link(i, Ri, pi);
    if constexpr (INV) {
      Sv<RC> a;
      if (fl & TDS_LF_PARENT_ADJ) a = a_prev_inv;
      else if (p >= 0) a = ld6<RC>(A.ptr<RC>(M.x_link + p * LWD), ST);
      else a = a_base_inv;
      Sv<RC> vJ; vJ.top = v3<RC>(RC(0), RC(0), RC(0)); vJ.bot = vJ.top;
      for (int c = 0; c < n_cols(i); ++c) {
        const Sv<RC> Sc = (fl & TDS_LF_SPHERICAL) ? S_col(i, c) : S;
        const RC qdc = qdv[(M.qd_idx[i] + c) * ST], qddc = qdd_in(M.qd_idx[i] + c);
        vJ.top = axpy(Sc.top, qdc, vJ.top); vJ.bot = axpy(Sc.bot, qdc, vJ.bot);
        a.top = axpy(Sc.top, qddc, a.top); a.bot = axpy(Sc.bot, qddc, a.bot);
      }
      a = a + cross_mm(v, vJ);                               // kinematics.hpp:96-97
      const Sv<RC> f = rbi_mul(r_inv, a) + cross_mf(v, rbi_mul(r_inv, v));
      for (int j = i; j >= 0; j = M.parent[j])               // the chain walk of crba_ancestors, from i itself
        for (int c = 0; c < n_cols(j); ++c) tauv[(M.qd_idx[j] + c) * ST] += dot(S_col(j, c), f);
      f_links = f_links + f;
      st6<RC>(A.ptr<RC>(M.x_link + i * LWD), ST, a);
      a_prev_inv = a;
    }
    // (REG also runs INV's statements above, the model's tau included, and never writes that tau: putting them under !REG reorders
    // four instructions of an existing INV instance)
    if constexpr (REG) reg_body(i + 1, i, Ri, pi, v, a_prev_inv, false);
    if constexpr (MOT) {   // a_i as INV carries it (a branch point's over its rigid-inertia words), then the outputs of the points on i
      Sv<RC> a;
      if (fl & TDS_LF_PARENT_ADJ) a = a_prev_inv;
      else if (p >= 0) a = ld6<RC>(A.ptr<RC>(M.x_link + p * LWD), ST);
      else a = a_base_inv;
      Sv<RC> vJ; vJ.top = v3<RC>(RC(0), RC(0), RC(0)); vJ.bot = vJ.top;
      for (int c = 0; c < n_cols(i); ++c) {
        const Sv<RC> Sc = (fl & TDS_LF_SPHERICAL) ? S_col(i, c) : S;
        const RC qdc = qdv[(M.qd_idx[i] + c) * ST], qddc = qdd_in(M.qd_idx[i] + c);
        vJ.top = axpy(Sc.top, qdc, vJ.top); vJ.bot = axpy(Sc.bot, qdc, vJ.bot);
        a.top = axpy(Sc.top, qddc, a.top); a.bot = axpy(Sc.bot, qddc, a.bot);
      }
      a = a + cross_mm(v, vJ);
      st6<RC>(A.ptr<RC>(M.x_link + i * LWD), ST, a);
      a_prev_inv = a;
      mot_link(i, Ri, pi, v, a);
    }
    if constexpr (DER) {   // a_i as INV carries it and f_i, kept in the derivative region
      Sv<RC> a;
      if (fl & TDS_LF_PARENT_ADJ) a = a_prev_inv;
      else if (p >= 0) a = ld6<RC>(derw + 12 * p * ST, ST);
      else a = a_base_inv;
      Sv<RC> vJ; vJ.top = v3<RC>(RC(0), RC(0), RC(0)); vJ.bot = vJ.top;
      for (int c = 0; c < n_cols(i); ++c) {
        const Sv<RC> Sc = S_col(i, c);
        const RC qdc = qdv[(M.qd_idx[i] + c) * ST], qddc = qdd_in(M.qd_idx[i] + c);
        vJ.top = axpy(Sc.top, qdc, vJ.top); vJ.bot = axpy(Sc.bot, qdc, vJ.bot);
        a.top = axpy(Sc.top, qddc, a.top); a.bot = axpy(Sc.bot, qddc, a.bot);
      }
      a = a + cross_mm(v, vJ);
      const Rbi<RC> r = ld_rbi<RC>(A.ptr<RC>(M.x_link + i * LWD), ST);
      st6<RC>(derw + 12 * i * ST, ST, a);
      st6<RC>(derw + (12 * i + 6) * ST, ST, rbi_mul(r, a) + cross_mf(v, rbi_mul(r, v)));
      a_prev_inv = a;
    }
    R_prev = Ri; p_prev = pi; v_prev = v;
  }
  if constexpr (KIN || MOT) return;
  if constexpr (REG) {
    // the base's columns: its own f in the base frame (rows 0..5) on a floating base, zero on a fixed one
    if (M.floating) {
      Sv<RC> vb, ab;
      vb.top = v3<RC>(qdv[0], qdv[ST], qdv[2 * ST]); vb.bot = v3<RC>(qdv[3 * ST], qdv[4 * ST], qdv[5 * ST]);
      ab.top = mulT(Rb, a_base_inv.top); ab.bot = mulT(Rb, a_base_inv.bot);
      reg_body(0, -1, m3_identity<RC>(), v3<RC>(RC(0), RC(0), RC(0)), vb, ab, true);
    } else {
      for (int c = 0; c < 10; ++c) {
        for (int k = 0; k < n; ++k) reg_put(io.jac, (size_t)k * n_pi + c, RC(0));
        reg_put(pm.yT, c, RC(0)); reg_put(pm.yV, c, RC(0));
      }
    }
    // stiffness (q, or a spherical joint's axis-angle vector) and damping (qd) columns of link i: nonzero in its own rows only
    for (int i = 0; i < n_links; ++i) {
      const int col = 10 * (n_links + 1) + 2 * i, nc = n_cols(i), d0 = M.qd_idx[i];
      RC sv[3] = {RC(0), RC(0), RC(0)};
      if (M.flags[i] & TDS_LF_SPHERICAL) { const V3<RC> aa = axis_angle(i); sv[0] = aa.x; sv[1] = aa.y; sv[2] = aa.z; }
      else if (nc > 0) sv[0] = qv[M.q_idx[i] * ST];
      RC vk = RC(0);
      for (int k = 0; k < n; ++k) {
        const bool own = nc > 0 && k >= d0 && k < d0 + nc;
        reg_put(io.jac, (size_t)k * n_pi + col, own ? sv[k - d0] : RC(0));
        reg_put(io.jac, (size_t)k * n_pi + col + 1, own ? RC(qdv[k * ST]) : RC(0));
      }
      for (int c = 0; c < nc; ++c) vk += sv[c] * sv[c];
      reg_put(pm.yT, col, RC(0)); reg_put(pm.yT, col + 1, RC(0));
      reg_put(pm.yV, col, RC(0.5) * vk); reg_put(pm.yV, col + 1, RC(0));
    }
    return;
  }
  if constexpr (INV) {
    for (int i = 0; i < n_links; ++i) {   // the stiffness and damping terms the ABA subtracts from tau
      const int fl = M.flags[i];
      if (fl & TDS_LF_FIXED) continue;
      const int d0 = M.qd_idx[i];
      if (fl & TDS_LF_SPHERICAL) {
        const RC d = joint_par(i, 1, M.damping[i]);
        for (int c = 0; c < 3; ++c) tauv[(d0 + c) * ST] += d * qdv[(d0 + c) * ST];
        if (M.stiffness[i] != 0.f || joint_slot(i, 0) >= 0) {
          const V3<RC> aa = axis_angle(i);
          const RC k = joint_par(i, 0, M.stiffness[i]);
          tauv[d0 * ST] += k * aa.x; tauv[(d0 + 1) * ST] += k * aa.y; tauv[(d0 + 2) * ST] += k * aa.z;
        }
      } else {
        tauv[d0 * ST] += joint_par(i, 0, M.stiffness[i]) * qv[M.q_idx[i] * ST] + joint_par(i, 1, M.damping[i]) * qdv[d0 * ST];
      }
    }
    if (M.floating) {   // the base's wrench [moment about the base origin; force] in the base frame
      Rbi<RC> Ib = model_rbi_of<RC>(M.base_rbi);
      if constexpr (PAR) { if (pm.any_base) installed_base(Ib); }
      Sv<RC> vb, ab;
      vb.top = v3<RC>(qdv[0], qdv[ST], qdv[2 * ST]); vb.bot = v3<RC>(qdv[3 * ST], qdv[4 * ST], qdv[5 * ST]);
      ab.top = mulT(Rb, a_base_inv.top); ab.bot = mulT(Rb, a_base_inv.bot);
      Sv<RC> fb = rbi_mul(Ib, ab) + cross_mf(vb, rbi_mul(Ib, vb));
      fb.top = fb.top + mulT(Rb, f_links.top); fb.bot = fb.bot + mulT(Rb, f_links.bot);
      tauv[0] += fb.top.x; tauv[ST] += fb.top.y; tauv[2 * ST] += fb.top.z;
      tauv[3 * ST] += fb.bot.x; tauv[4 * ST] += fb.bot.y; tauv[5 * ST] += fb.bot.z;
    }
    if (live && io.jac)
      for (int k = 0; k < n; ++k) {
        if constexpr (AD) io.jac[((size_t)k * io.jac_n_in + jcol) * ns + e] = tauv[k * ST].d;
        else io.jac[(size_t)k * ns + e] = tauv[k * ST];
      }
    return;
  }
  // CEN: the centre of mass relative to O; row r of an output; column col of A from the momentum F about O of qd_col = 1: [k_O - c x l; l]
  typename std::conditional<CEN, V3<RC>, NoPar>::type cen_c{};
  if constexpr (CEN) cen_c = cen_I.h * (RC(1) / cen_I.m);
  auto cen_put = [&](double* o, size_t r, const RC& x) {
    if constexpr (CEN) {
      if (!o || !live) return;
      if constexpr (AD) o[(r * io.jac_n_in + jcol) * ns + e] = x.d;
      else o[r * ns + e] = x;
    }
  };
  auto cen_col = [&](int col, const Sv<RC>& F) {
    if constexpr (CEN) {
      const V3<RC> k = F.top - cross(cen_c, F.bot);
      cen_put(pm.A, col, k.x); cen_put(pm.A, n + col, k.y); cen_put(pm.A, 2 * n + col, k.z);
      cen_put(pm.A, 3 * n + col, F.bot.x); cen_put(pm.A, 4 * n + col, F.bot.y); cen_put(pm.A, 5 * n + col, F.bot.z);
    }
  };
  // ---- contacts between the multibodies of the world (world.hpp:206-282), group = ordered pair of multibodies -----------------------
  // contact_sphere_sphere (contact_point.hpp:44-94) on sphere centres / capsule end spheres (contact_capsule_sphere, :406-438);
  // sphere A x capsule B goes through the dispatcher's swapped call (:478-492): points exchanged, normal negated.
  // Record: point on a [3] (relative to O), normal on b [3], distance, link a, link b; point on b = point on a - distance * normal.
  int pgc[TDS_MAX_PAIR_GROUPS];
  int n_pair_active = 0;
  if (want_contacts && M.n_pair_points > 0) {
    for (int g = 0; g < M.n_pair_groups; ++g) {
      int cnt = 0;
      for (int pt = M.pg_begin[g]; pt < M.pg_begin[g + 1]; ++pt) {
        const int ga = M.pp_ga[pt], gb = M.pp_gb[pt], kind = M.pp_kind[pt];
        const RC* wa = A.ptr<RC>(M.x_gw + M.g_wslot[ga] * 12 * RCW);
        const RC* wb = A.ptr<RC>(M.x_gw + M.g_wslot[gb] * 12 * RCW);
        if (kind >= 100) {
          // a PLANE shape on a link x point k of the other multibody's sphere / capsule / box: contact_plane_sphere
          // (contact_point.hpp:97-124) on the sphere, the capsule's end spheres (+L/2, -L/2) or the box's corner spheres (x outermost);
          // plane constant 0, world-frame normal as given - the pose of the plane's link is not used; a point is always emitted
          const bool swapped = kind >= 200;                      // the plane is on b: points exchanged, normal negated (:478-492)
          const int gp = swapped ? gb : ga, go = swapped ? ga : gb, k = kind - (swapped ? 200 : 100);
          const RC* wo = swapped ? wa : wb;
          const V3<RC> pnrm = v3<RC>(RC(M.g_half[gp][0]), RC(M.g_half[gp][1]), RC(M.g_half[gp][2]));
          V3<RC> c = ld3<RC>(wo, ST);
          const int to = M.g_type[go];
          if (to == TDSG_CAPSULE) c = k == 0 ? c + ld3<RC>(wo + 3 * ST, ST) : c - ld3<RC>(wo + 3 * ST, ST);
          else if (to == TDSG_BOX) {
            const V3<RC> ex = ld3<RC>(wo + 3 * ST, ST), ey = ld3<RC>(wo + 6 * ST, ST), ez = ld3<RC>(wo + 9 * ST, ST);
            c = (k & 4) ? c - ex : c + ex;
            c = (k & 2) ? c - ey : c + ey;
            c = (k & 1) ? c - ez : c + ez;
          }
          const RC rad = RC(M.g_radius[go]);
          const RC t = dot(c + O, pnrm);                         // -(dot(position, -normal) + constant), constant = 0
          const RC dist = t - rad;
          if (io.contact_dist && live) io.contact_dist[(size_t)(pt_index + pt) * ns + e] = (float)val_of(dist);
          if constexpr (CF) {   // point on b: on the sphere (the plane on a), else on the plane
            if (!swapped) cf_geom(pt_index + pt, v3<RC>(-pnrm.x, -pnrm.y, -pnrm.z), c - pnrm * rad, dist);
            else cf_geom(pt_index + pt, pnrm, c - pnrm * t, dist);
            if (dist < RC(0)) cf_pair |= 1ull << pt;
          }
          if (dist < RC(0)) {
            RC* pr = A.ptr<RC>(M.x_pcon + n_pair_active * 9 * RCW);
            if (!swapped) { st3<RC>(pr, ST, c - pnrm * t); st3<RC>(pr + 3 * ST, ST, v3<RC>(-pnrm.x, -pnrm.y, -pnrm.z)); }   // point on the plane, normal on b = -n
            else { st3<RC>(pr, ST, c - pnrm * rad); st3<RC>(pr + 3 * ST, ST, pnrm); }                                        // point on the sphere, normal = +n
            pr[6 * ST] = dist;
            pr[7 * ST] = RC(M.g_link[ga]);
            pr[8 * ST] = RC(M.g_link[gb]);
            ++n_pair_active; ++cnt;
          }
          continue;
        }
        V3<RC> ca = ld3<RC>(wa, ST), cb = ld3<RC>(wb, ST);
        if (kind == 1) ca = ca + ld3<RC>(wa + 3 * ST, ST); else if (kind == -1) ca = ca - ld3<RC>(wa + 3 * ST, ST);
        if (kind == 2) cb = cb + ld3<RC>(wb + 3 * ST, ST); else if (kind == -2) cb = cb - ld3<RC>(wb + 3 * ST, ST);
        const bool swapped = kind == 2 || kind == -2;          // the contact function ran with (capsule on b, sphere on a)
        const RC r1 = RC(swapped ? M.g_radius[gb] : M.g_radius[ga]), r2 = RC(swapped ? M.g_radius[ga] : M.g_radius[gb]);
        const V3<RC> diff = swapped ? cb - ca : ca - cb;       // poseA.position - poseB.position of the call
        const RC len = sqrt_t(dot(diff, diff));
        const RC dist = len - (r1 + r2);
        // candidate distances behind the plane candidates; +inf: the contact function emitted no point (centres closer than CONTACT_EPSILON)
        if (io.contact_dist && live) io.contact_dist[(size_t)(pt_index + pt) * ns + e] = len > RC(1e-5) ? (float)val_of(dist) : __int_as_float(0x7f800000);
        if constexpr (CF) {   // the record's point on b and normal on b, as stored below; no point emitted: zeros and distance +inf
          if (len > RC(1e-5)) {
            const V3<RC> nrm = diff * (RC(1) / len);
            const V3<RC> p1 = (swapped ? cb : ca) - nrm * r1;
            if (swapped) cf_geom(pt_index + pt, v3<RC>(-nrm.x, -nrm.y, -nrm.z), p1, dist);
            else cf_geom(pt_index + pt, nrm, p1 - nrm * dist, dist);
          } else {
            const V3<RC> z = v3<RC>(RC(0), RC(0), RC(0));
            cf_geom(pt_index + pt, z, z, RC(__int_as_float(0x7f800000)));
            for (int r = 3; r < 6; ++r) cf_put(10 * (pt_index + pt) + r, RC(0));   // (cf_geom adds O)
          }
          if (len > RC(1e-5) && dist < RC(0)) cf_pair |= 1ull << pt;
        }
        if (len > RC(1e-5) && dist < RC(0)) {                  // CONTACT_EPSILON; resolve_collision keeps distance < 0 (the others are zero rows)
          const V3<RC> nrm = diff * (RC(1) / len);
          const V3<RC> p1 = (swapped ? cb : ca) - nrm * r1;    // point_a_world of the call
          RC* pr = A.ptr<RC>(M.x_pcon + n_pair_active * 9 * RCW);
          if (swapped) { st3<RC>(pr, ST, p1 - nrm * dist); st3<RC>(pr + 3 * ST, ST, v3<RC>(-nrm.x, -nrm.y, -nrm.z)); }
          else { st3<RC>(pr, ST, p1); st3<RC>(pr + 3 * ST, ST, nrm); }
          pr[6 * ST] = dist;
          pr[7 * ST] = RC(M.g_link[ga]);
          pr[8 * ST] = RC(M.g_link[gb]);
          ++n_pair_active; ++cnt;
        }
      }
      pgc[g] = cnt;
    }
  }
  const bool any_contact = MASS || __any_sync(0xffffffffu, n_active > 0 || n_pair_active > 0);   // MASS: the CRBA always runs
  TDSW_PHASE();  // 2

  // ---- pass 2: leaf -> root.  ABA (forward_dynamics.hpp:50-216) + CRBA (mass_matrix.hpp:39-125) ----------
  if (any_contact) {
    const int nblk = nb * (nb + 1) / 2 * 9;
    for (int k = 0; k < nblk; ++k) Mb[k * ST] = RS(0);
    for (int k = n; k < n3; ++k) Mb[(btri(k / 3, k / 3) + (k % 3) * 4) * ST] = RS(1);   // padding dofs: identity
  }
  Abi<RA> cA; Sv<RA> cP; Rbi<RC> cC;
  // M(r, c) = S_c . F for every dof column c of the ancestors of link i (and of the floating base), F = Ic S_r
  // (mass_matrix.hpp:58-111); r > c always: links are ordered parent first
  auto Mset = [&](int r, int c, RS val) { Mb[(btri(r / 3, c / 3) + (r % 3) * 3 + (c % 3)) * ST] = val; };
  auto crba_ancestors = [&](int i, int row, const Sv<RC>& F) {
    for (int j = M.parent[i]; j >= 0; j = M.parent[j]) {
      const int nc = n_cols(j);
      for (int c = 0; c < nc; ++c) Mset(row, M.qd_idx[j] + c, RS(dot(S_col(j, c), F)));
    }
    if (M.floating) {  // base columns: F in the base frame (:107-111); O is the base origin
      const V3<RC> ft = mulT(Rb, F.top), fb = mulT(Rb, F.bot);
      Mset(row, 0, RS(ft.x)); Mset(row, 1, RS(ft.y)); Mset(row, 2, RS(ft.z));
      Mset(row, 3, RS(fb.x)); Mset(row, 4, RS(fb.y)); Mset(row, 5, RS(fb.z));
    }
  };
  // Ia -= a b^T in the block form of the 1-dof update below (I: top-top, H: top-bot, M: bot-bot)
  auto abi_sub_outer = [&](Abi<RA>& Ia, const Sv<RA>& a, const Sv<RA>& b) {
    Ia.I.xx -= a.top.x * b.top.x; Ia.I.xy -= a.top.x * b.top.y; Ia.I.xz -= a.top.x * b.top.z;
    Ia.I.yy -= a.top.y * b.top.y; Ia.I.yz -= a.top.y * b.top.z; Ia.I.zz -= a.top.z * b.top.z;
    Ia.H.xx -= a.top.x * b.bot.x; Ia.H.xy -= a.top.x * b.bot.y; Ia.H.xz -= a.top.x * b.bot.z;
    Ia.H.yx -= a.top.y * b.bot.x; Ia.H.yy -= a.top.y * b.bot.y; Ia.H.yz -= a.top.y * b.bot.z;
    Ia.H.zx -= a.top.z * b.bot.x; Ia.H.zy -= a.top.z * b.bot.y; Ia.H.zz -= a.top.z * b.bot.z;
    Ia.M.xx -= a.bot.x * b.bot.x; Ia.M.xy -= a.bot.x * b.bot.y; Ia.M.xz -= a.bot.x * b.bot.z;
    Ia.M.yy -= a.bot.y * b.bot.y; Ia.M.yz -= a.bot.y * b.bot.z; Ia.M.zz -= a.bot.z * b.bot.z;
  };
  // COR: entry k of C; the rate r' of a rigid inertia r about O moving with v = [w; u]: h' = m u + w x h, I' = [w]x I - I [w]x +
  // 2 (h . u) 1 - u h^T - h u^T; B u and B^T u of the composites (D = Ic', h); the composites handed from an adjacent child
  auto cor_put = [&](int k, const RC& x) {
    if constexpr (COR) {
      if (!live || !io.jac) return;
      if constexpr (AD) io.jac[((size_t)k * io.jac_n_in + jcol) * ns + e] = x.d;
      else io.jac[(size_t)k * ns + e] = x;
    }
  };
  auto cor_rate = [&](const Rbi<RC>& r, const Sv<RC>& v) -> Rbi<RC> {
    Rbi<RC> o;
    const V3<RC> w = v.top, u = v.bot;
    o.m = RC(0);
    o.h = u * r.m + cross(w, r.h);
    const V3<RC> a0 = cross(w, v3<RC>(r.I.xx, r.I.xy, r.I.xz)), a1 = cross(w, v3<RC>(r.I.xy, r.I.yy, r.I.yz)),
                 a2 = cross(w, v3<RC>(r.I.xz, r.I.yz, r.I.zz));   // the columns of [w]x I
    const RC hu = dot(r.h, u);
    o.I.xx = RC(2) * (a0.x + hu - u.x * r.h.x); o.I.yy = RC(2) * (a1.y + hu - u.y * r.h.y); o.I.zz = RC(2) * (a2.z + hu - u.z * r.h.z);
    o.I.xy = a1.x + a0.y - u.x * r.h.y - r.h.x * u.y;
    o.I.xz = a2.x + a0.z - u.x * r.h.z - r.h.x * u.z;
    o.I.yz = a2.y + a1.z - u.y * r.h.z - r.h.y * u.z;
    return o;
  };
  auto cor_B = [&](const Rbi<RC>& D, const Sv<RC>& h, const Sv<RC>& u, bool transposed) -> Sv<RC> {
    const Sv<RC> a = rbi_mul(D, u), b = cross_mf(u, h);
    const RC s = transposed ? RC(-0.5) : RC(0.5);
    Sv<RC> o;
    o.top = a.top * RC(0.5) + b.top * s;
    o.bot = a.bot * RC(0.5) + b.bot * s;
    return o;
  };
  typename std::conditional<COR || DER, Rbi<RC>, NoPar>::type cor_cD{};
  typename std::conditional<COR || DER, Sv<RC>, NoPar>::type cor_cH{};
  if constexpr (COR) {
    static_assert(std::is_same<RA, RC>::value && std::is_same<RC, RQ>::value, "the COR instances run in one scalar type");
    for (int k = 0; k < n * n; ++k) cor_put(k, RC(0));
  }
  // DER: entry k of d tau / dq (o = 0) or d tau / dqd (o = 1); the subtree force handed from an adjacent child; column c of link j (-1:
  // the floating base's twist column c) with the quantities that do not move with the subtree (see the comment on the kernel)
  auto der_put = [&](int o, int k, const RC& x) {
    if constexpr (DER) {
      double* out = o ? io.g_in : io.jac;
      if (!live || !out) return;
      if constexpr (AD) out[((size_t)k * io.jac_n_in + jcol) * ns + e] = x.d;
      else out[(size_t)k * ns + e] = x;
    }
  };
  typename std::conditional<DER, Sv<RC>, NoPar>::type der_cF{};
  auto der_col = [&](int j, int c, Sv<RC>& S, Sv<RC>& al, Sv<RC>& ga, Sv<RC>& ps) {
    if constexpr (DER) {
      const Sv<RC> z = Sv<RC>{v3<RC>(RC(0), RC(0), RC(0)), v3<RC>(RC(0), RC(0), RC(0))};
      Sv<RC> vl = z, al_ = z, vj = v_base;   // the base's: the world's velocity and acceleration (-g)
      al_.bot = v3<RC>(RC(-P.gravity[0]), RC(-P.gravity[1]), RC(-P.gravity[2]));
      if (j >= 0) {
        const int pj = M.parent[j];
        if (pj >= 0) { vl = ld6<RC>(A.ptr<RC>(M.x_link + pj * LWD + VOFF), ST); al_ = ld6<RC>(derw + 12 * pj * ST, ST); }
        else { vl = v_base; al_ = a_base_inv; }
        vj = ld6<RC>(A.ptr<RC>(M.x_link + j * LWD + VOFF), ST);
        S = S_col(j, c);
      } else {
        const V3<RC> u = c % 3 == 0 ? col_x(Rb) : (c % 3 == 1 ? col_y(Rb) : col_z(Rb));
        S = z;
        if (c < 3) S.top = u; else S.bot = u;
      }
      al = cross_mm(vl, S);
      ga = cross_mm(al_, S) + cross_mm(vl, al);
      ps = cross_mm(vl + vj, S);
    }
  };
  if constexpr (DER) {
    for (int k = 0; k < n * n; ++k) { der_put(0, k, RC(0)); der_put(1, k, RC(0)); }
  }
  for (int i = n_links - 1; i >= 0; --i) {
    const int p = M.parent[i];
    const int fl = M.flags[i];
    RC* const rec = A.ptr<RC>(M.x_link + i * LWD);
    RA* const vrec = A.ptr<RA>(M.x_link + i * LWD + VOFF);
    Rbi<RC> Ic = ld_rbi<RC>(rec, ST);
    const Rbi<RA> rb = cvt_rbi<RA>(Ic);
    const Sv<RA> v = ld6<RA>(vrec, ST);
    Abi<RA> Ia = abi_from_rbi(rb);
    Sv<RA> pA = cross_mf(v, rbi_mul(rb, v));                 // kinematics.hpp:132
    if constexpr (EXT) {                                     // - f_ext, the sum pass 1 stored
      if ((pm.ext.links_with_points >> i) & 1ull) {
        const Sv<RA> w = ld6<RA>(A.ptr<RA>(pm.ext.x_ext + i * 6 * RAW), ST);
        pA.top = pA.top - w.top; pA.bot = pA.bot - w.bot;
      }
    }
    // COR: the link's own rate and momentum, then its children's composites (in the accumulators' ABA words: rate 10, momentum 6)
    // DER: these and the subtree force (rate 10, momentum 6, force 6)
    typename std::conditional<COR || DER, Rbi<RC>, NoPar>::type cor_D{};
    typename std::conditional<COR || DER, Sv<RC>, NoPar>::type cor_h{};
    typename std::conditional<DER, Sv<RC>, NoPar>::type der_F{};
    if constexpr (COR || DER) { cor_D = cor_rate(Ic, v); cor_h = rbi_mul(Ic, v); }
    if constexpr (DER) der_F = ld6<RC>(derw + (12 * i + 6) * ST, ST);
    if (fl & TDS_LF_CHILD_ADJ) {
      if constexpr (!MASS && !CEN && !COR && !DER) { abi_add(Ia, cA); pA = pA + cP; }
      rbi_add(Ic, cC);
      if constexpr (COR || DER) { rbi_add(cor_D, cor_cD); cor_h = cor_h + cor_cH; }
      if constexpr (DER) der_F = der_F + der_cF;
    }
    if (M.acc_slot[i] >= 0) {
      if constexpr (!MASS && !CEN && !COR && !DER) {
        Abi<RA> sa; Sv<RA> sp;
        acc_ld27<RA>(A.ptr<RA>(M.x_acc + M.acc_slot[i] * M.x_acc_words), ST, sa, sp);
        abi_add(Ia, sa); pA = pA + sp;
      }
      rbi_add(Ic, ld_rbi<RC>(A.ptr<RC>(M.x_acc + M.acc_slot[i] * M.x_acc_words + M.x_acc_ic_word), ST));
      if constexpr (COR || DER) {
        const RC* pc = A.ptr<RC>(M.x_acc + M.acc_slot[i] * M.x_acc_words);
        rbi_add(cor_D, ld_rbi<RC>(pc, ST));
        cor_h = cor_h + ld6<RC>(pc + 10 * ST, ST);
        if constexpr (DER) der_F = der_F + ld6<RC>(pc + 16 * ST, ST);
      }
    }
    Sv<RA> pa = pA;
    // U (6), invD, u overwrite the rigid-inertia record.  The RA and RC views interleave lanes differently, so
    // every lane must have finished reading its RC record before any lane writes the RA view.
    __syncwarp();
    RA* const urec = A.ptr<RA>(M.x_link + i * LWD);
    if constexpr (CEN) {   // the columns of link i's dofs, F = Ic S; Ic (v x S qd) into the rate (Ic c summed over links = sum r a)
      Sv<RC> vJ; vJ.top = v3<RC>(RC(0), RC(0), RC(0)); vJ.bot = vJ.top;
      for (int a = 0; a < n_cols(i); ++a) {
        const Sv<RC> Sc = S_col(i, a);
        const RC qda = qdv[(M.qd_idx[i] + a) * ST];
        vJ.top = axpy(Sc.top, qda, vJ.top); vJ.bot = axpy(Sc.bot, qda, vJ.bot);
        cen_col(M.qd_idx[i] + a, rbi_mul(Ic, Sc));
      }
      cen_f = cen_f + rbi_mul(Ic, cross_mm(v, vJ));
    } else if constexpr (MASS) {   // the CRBA columns of the two branches below (mass_matrix.hpp:58-111), without the ABA
      const int d0 = M.qd_idx[i];
      for (int a = 0; a < n_cols(i); ++a) {
        const Sv<RC> F = rbi_mul(Ic, S_col(i, a));
        for (int b = 0; b <= a; ++b) Mset(d0 + a, d0 + b, RS(dot(S_col(i, b), F)));
        crba_ancestors(i, d0 + a, F);
      }
    } else if constexpr (COR) {   // C's entries between link i's dofs and those of i and its ancestors, column a of i at a time
      const int d0 = M.qd_idx[i], nc = n_cols(i);
      for (int a = 0; a < nc; ++a) {
        const Sv<RC> S = S_col(i, a);
        const Sv<RC> G = rbi_mul(Ic, S), Hs = cor_B(cor_D, cor_h, S, true);   // Ic S_a, B^T S_a
        const Sv<RC> F = rbi_mul(Ic, cross_mm(v, S)) + cor_B(cor_D, cor_h, S, false);
        for (int b = 0; b < nc; ++b) cor_put((d0 + b) * n + d0 + a, dot(S_col(i, b), F));
        for (int j = M.parent[i]; j >= 0; j = M.parent[j]) {
          const int ncj = n_cols(j);
          if (ncj == 0) continue;
          const Sv<RC> Y = cross_mf(ld6<RC>(A.ptr<RC>(M.x_link + j * LWD + VOFF), ST), G);
          Sv<RC> X; X.top = Hs.top - Y.top; X.bot = Hs.bot - Y.bot;   // G_a . (v_j x S_b) = -(v_j x* G_a) . S_b
          for (int b = 0; b < ncj; ++b) {
            const Sv<RC> Sb = S_col(j, b);
            cor_put((d0 + a) * n + M.qd_idx[j] + b, dot(X, Sb));
            cor_put((M.qd_idx[j] + b) * n + d0 + a, dot(Sb, F));
          }
        }
        if (M.floating) {   // the base twist's columns [R_b e_k; 0], [0; R_b e_k]: a dot product with one is a base-frame component
          const Sv<RC> Y = cross_mf(v_base, G);
          const V3<RC> xt = mulT(Rb, Hs.top - Y.top), xb = mulT(Rb, Hs.bot - Y.bot);
          const V3<RC> ft = mulT(Rb, F.top), fb = mulT(Rb, F.bot);
          const int r = (d0 + a) * n;
          cor_put(r, xt.x); cor_put(r + 1, xt.y); cor_put(r + 2, xt.z); cor_put(r + 3, xb.x); cor_put(r + 4, xb.y); cor_put(r + 5, xb.z);
          cor_put(d0 + a, ft.x); cor_put(n + d0 + a, ft.y); cor_put(2 * n + d0 + a, ft.z);
          cor_put(3 * n + d0 + a, fb.x); cor_put(4 * n + d0 + a, fb.y); cor_put(5 * n + d0 + a, fb.z);
        }
      }
    } else if constexpr (DER) {   // link i's rows and columns against those of i and its ancestors, column a of i at a time
      const int d0 = M.qd_idx[i], nc = n_cols(i);
      for (int a = 0; a < nc; ++a) {
        Sv<RC> S, al, ga, ps;
        der_col(i, a, S, al, ga, ps);
        const Sv<RC> G = rbi_mul(Ic, S), Sh = cross_mf(S, cor_h);
        Sv<RC> H = rbi_mul(cor_D, S);   // row a against a column: (Ic S_a) . gamma + H . alpha
        H.top = H.top - Sh.top; H.bot = H.bot - Sh.bot;
        const Sv<RC> Fn = rbi_mul(Ic, ga) + rbi_mul(cor_D, al) + cross_mf(al, cor_h);
        const Sv<RC> Fd = rbi_mul(Ic, ps) + rbi_mul(cor_D, S) + cross_mf(S, cor_h);
        const Sv<RC> Fq = Fn + cross_mf(S, der_F);
        for (int b = 0; b < nc; ++b) {
          const Sv<RC> Sb = S_col(i, b);
          RC kq = RC(0), kd = RC(0);   // the stiffness and damping terms
          if (fl & TDS_LF_SPHERICAL) {
            if (a == b) kd = joint_par(i, 1, M.damping[i]);
            if (M.stiffness[i] != 0.f || joint_slot(i, 0) >= 0) {   // d/de axis_angle(q (+) e e_a), q' = 1/2 q (x) (e_a, 0)
              typedef tds::Dual<RC> T;
              const int q0 = M.q_idx[i];
              const RC x = qv[q0 * ST], y = qv[(q0 + 1) * ST], z = qv[(q0 + 2) * ST], w = qv[(q0 + 3) * ST];
              const V3<RC> ea = v3<RC>(RC(a == 0), RC(a == 1), RC(a == 2));
              const V3<RC> dv = (ea * w + cross(v3<RC>(x, y, z), ea)) * RC(0.5);
              const V3<T> aa = axis_angle_of(T(x, dv.x), T(y, dv.y), T(z, dv.z), T(w, RC(-0.5) * dot(v3<RC>(x, y, z), ea)));
              kq = joint_par(i, 0, M.stiffness[i]) * (b == 0 ? aa.x : (b == 1 ? aa.y : aa.z)).d;
            }
          } else {
            kd = joint_par(i, 1, M.damping[i]);
            kq = joint_par(i, 0, M.stiffness[i]);
            if (M.jtype[i] == TDSJ_REVOLUTE_AXIS && !(fl & TDS_LF_PRISMATIC)) {   // q' = |axis| along the unit tangent
              const V3<RC> ax = v3<RC>(RC(M.axis[i][0]), RC(M.axis[i][1]), RC(M.axis[i][2]));
              kq = kq * sqrt_t(dot(ax, ax));
            }
          }
          der_put(0, (d0 + b) * n + d0 + a, dot(Sb, Fn) + kq);
          der_put(1, (d0 + b) * n + d0 + a, dot(Sb, Fd) + kd);
        }
        for (int j = M.parent[i]; j >= 0; j = M.parent[j]) {
          for (int b = 0; b < n_cols(j); ++b) {
            Sv<RC> Sb, alb, gab, psb;
            der_col(j, b, Sb, alb, gab, psb);
            const int rj = M.qd_idx[j] + b;
            der_put(0, rj * n + d0 + a, dot(Sb, Fq));
            der_put(1, rj * n + d0 + a, dot(Sb, Fd));
            der_put(0, (d0 + a) * n + rj, dot(G, gab) + dot(H, alb));
            der_put(1, (d0 + a) * n + rj, dot(G, psb) + dot(H, Sb));
          }
        }
        if (M.floating) {   // the base twist's columns: a dot product with one is a base-frame component
          const V3<RC> qt = mulT(Rb, Fq.top), qb = mulT(Rb, Fq.bot), dt = mulT(Rb, Fd.top), db = mulT(Rb, Fd.bot);
          const RC fq[6] = {qt.x, qt.y, qt.z, qb.x, qb.y, qb.z}, fd[6] = {dt.x, dt.y, dt.z, db.x, db.y, db.z};
          for (int k = 0; k < 6; ++k) {
            Sv<RC> Sb, alb, gab, psb;
            der_col(-1, k, Sb, alb, gab, psb);
            der_put(0, k * n + d0 + a, fq[k]);
            der_put(1, k * n + d0 + a, fd[k]);
            der_put(0, (d0 + a) * n + k, dot(G, gab));
            der_put(1, (d0 + a) * n + k, dot(G, psb) + dot(H, Sb));
          }
        }
      }
    } else if (fl & TDS_LF_FIXED) {
      Sv<RA> z; z.top = v3<RA>(RA(0), RA(0), RA(0)); z.bot = z.top;
      st6<RA>(vrec, ST, z);
      st6<RA>(urec, ST, z);
      urec[6 * ST] = RA(0); urec[7 * ST] = RA(0);
    } else if (fl & TDS_LF_SPHERICAL) {
      // 3-dof joint (forward_dynamics.hpp:56-109): U = Ia S, D = S^T U (3 x 3), u = tau - damping qd - S^T pA,
      // Ia -= U D^-1 U^T, pa = pA + Ia c + U D^-1 u.  Record: U (18) | D^-1 (9) | u (3), then c.
      const int d0 = M.qd_idx[i];
      Sv<RC> Sd[3]; Sv<RA> S[3], U[3];
      RA qdj[3];
      Sv<RA> vJ; vJ.top = v3<RA>(RA(0), RA(0), RA(0)); vJ.bot = vJ.top;
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        Sd[a] = S_col(i, a); S[a] = cvt_sv<RA>(Sd[a]);
        qdj[a] = RA(qdv[(d0 + a) * ST]);
        vJ.top = axpy(S[a].top, qdj[a], vJ.top); vJ.bot = axpy(S[a].bot, qdj[a], vJ.bot);
        U[a] = abi_mul(Ia, S[a]);
      }
      const Sv<RA> c = cross_mm(v, vJ);                      // kinematics.hpp:96-97
      RA Dm[3][3], u[3];
#pragma unroll
      for (int a = 0; a < 3; ++a) {
#pragma unroll
        for (int b = 0; b < 3; ++b) Dm[a][b] = dot(S[a], U[b]);
        u[a] = RA(tauv[(d0 + a) * ST]) - RA(joint_par(i, 1, M.damping[i])) * qdj[a] - dot(S[a], pA);
      }
      // (an installed stiffness always takes this path: its derivative at 0 is not lost)
      if (M.stiffness[i] != 0.f || joint_slot(i, 0) >= 0) {   // tau -= stiffness * quaternion_axis_angle(q), forward_dynamics.hpp:69-74, tiny_algebra.hpp:509-527
        const int q0 = M.q_idx[i];
        const RC qx = RC(qv[q0 * ST]), qy = RC(qv[(q0 + 1) * ST]), qz = RC(qv[(q0 + 2) * ST]), qw = RC(qv[(q0 + 3) * ST]);
        const RC nrm = sqrt_t(qx * qx + qy * qy + qz * qz);
        const RC theta = RC(2) * atan2_t(nrm, qw);
        const RC scaling = nrm < RC(1.220703125e-4) ? RC(1) / (RC(0.5) + theta * theta * RC(1.0 / 48.0)) : theta / nrm;   // eps^(1/4)
        const RA k = RA(joint_par(i, 0, M.stiffness[i]));
        u[0] -= k * RA(scaling * qx); u[1] -= k * RA(scaling * qy); u[2] -= k * RA(scaling * qz);
      }
      RA Di[3][3];   // general 3 x 3 inverse (Matrix3::inverse)
      {
        const RA c0 = Dm[1][1] * Dm[2][2] - Dm[1][2] * Dm[2][1], c1 = Dm[1][2] * Dm[2][0] - Dm[1][0] * Dm[2][2], c2 = Dm[1][0] * Dm[2][1] - Dm[1][1] * Dm[2][0];
        const RA sdet = RA(1) / (Dm[0][0] * c0 + Dm[0][1] * c1 + Dm[0][2] * c2);
        Di[0][0] = c0 * sdet; Di[0][1] = (Dm[0][2] * Dm[2][1] - Dm[0][1] * Dm[2][2]) * sdet; Di[0][2] = (Dm[0][1] * Dm[1][2] - Dm[0][2] * Dm[1][1]) * sdet;
        Di[1][0] = c1 * sdet; Di[1][1] = (Dm[0][0] * Dm[2][2] - Dm[0][2] * Dm[2][0]) * sdet; Di[1][2] = (Dm[0][2] * Dm[1][0] - Dm[0][0] * Dm[1][2]) * sdet;
        Di[2][0] = c2 * sdet; Di[2][1] = (Dm[0][1] * Dm[2][0] - Dm[0][0] * Dm[2][1]) * sdet; Di[2][2] = (Dm[0][0] * Dm[1][1] - Dm[0][1] * Dm[1][0]) * sdet;
      }
      st6<RA>(vrec, ST, c);
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        st6<RA>(urec + a * 6 * ST, ST, U[a]);
#pragma unroll
        for (int b = 0; b < 3; ++b) urec[(18 + a * 3 + b) * ST] = Di[a][b];
        urec[(27 + a) * ST] = u[a];
      }
      Sv<RA> V[3];   // V = U D^-1
#pragma unroll
      for (int b = 0; b < 3; ++b) {
        V[b].top = U[0].top * Di[0][b] + U[1].top * Di[1][b] + U[2].top * Di[2][b];
        V[b].bot = U[0].bot * Di[0][b] + U[1].bot * Di[1][b] + U[2].bot * Di[2][b];
      }
#pragma unroll
      for (int b = 0; b < 3; ++b) abi_sub_outer(Ia, V[b], U[b]);
      const Sv<RA> Iac = abi_mul(Ia, c);
      pa.top = pA.top + Iac.top + V[0].top * u[0] + V[1].top * u[1] + V[2].top * u[2];
      pa.bot = pA.bot + Iac.bot + V[0].bot * u[0] + V[1].bot * u[1] + V[2].bot * u[2];
      if (any_contact) {   // mass_matrix.hpp:58-84
#pragma unroll
        for (int a = 0; a < 3; ++a) {
          const Sv<RC> F = rbi_mul(Ic, Sd[a]);
          for (int b = 0; b <= a; ++b) Mset(d0 + a, d0 + b, RS(dot(Sd[b], F)));
          crba_ancestors(i, d0 + a, F);
        }
      }
    } else {
      const Sv<RC> Sd = ld6<RC>(Sw + i * 6 * ST, ST);
      const Sv<RA> S = cvt_sv<RA>(Sd);
      const int qdi = M.qd_idx[i];
      const RA qdj = RA(qdv[qdi * ST]);
      Sv<RA> vJ; vJ.top = S.top * qdj; vJ.bot = S.bot * qdj;
      const Sv<RA> c = cross_mm(v, vJ);                      // kinematics.hpp:96-97
      const Sv<RA> U = abi_mul(Ia, S);                       // forward_dynamics.hpp:111
      const RA D = dot(S, U);
      const RA invD = RA(1) / D;
      RA tau = RA(tauv[qdi * ST]);
      tau -= RA(joint_par(i, 0, M.stiffness[i])) * RA(qv[M.q_idx[i] * ST]);
      tau -= RA(joint_par(i, 1, M.damping[i])) * qdj;
      const RA u = tau - dot(S, pA);                         // :129
      st6<RA>(vrec, ST, c);
      st6<RA>(urec, ST, U);
      urec[6 * ST] = invD; urec[7 * ST] = u;
      const V3<RA> ut = U.top * invD, ub = U.bot * invD;     // Ia -= U (U/D)^T, :160-168
      Ia.I.xx -= U.top.x * ut.x; Ia.I.xy -= U.top.x * ut.y; Ia.I.xz -= U.top.x * ut.z;
      Ia.I.yy -= U.top.y * ut.y; Ia.I.yz -= U.top.y * ut.z; Ia.I.zz -= U.top.z * ut.z;
      Ia.H.xx -= U.top.x * ub.x; Ia.H.xy -= U.top.x * ub.y; Ia.H.xz -= U.top.x * ub.z;
      Ia.H.yx -= U.top.y * ub.x; Ia.H.yy -= U.top.y * ub.y; Ia.H.yz -= U.top.y * ub.z;
      Ia.H.zx -= U.top.z * ub.x; Ia.H.zy -= U.top.z * ub.y; Ia.H.zz -= U.top.z * ub.z;
      Ia.M.xx -= U.bot.x * ub.x; Ia.M.xy -= U.bot.x * ub.y; Ia.M.xz -= U.bot.x * ub.z;
      Ia.M.yy -= U.bot.y * ub.y; Ia.M.yz -= U.bot.y * ub.z; Ia.M.zz -= U.bot.z * ub.z;
      const Sv<RA> Iac = abi_mul(Ia, c);                     // :171
      const RA uD = u * invD;
      pa.top = pA.top + Iac.top + U.top * uD;                // :173
      pa.bot = pA.bot + Iac.bot + U.bot * uD;
      if (any_contact) {   // CRBA column, mass_matrix.hpp:86-111: M_ij = S_j . (Ic_i S_i), no transforms needed
        const Sv<RC> F = rbi_mul(Ic, Sd);
        Mset(qdi, qdi, RS(dot(Sd, F)));
        crba_ancestors(i, qdi, F);
      }
    }
    // hand (Ia, pa, Ic) to the parent: plain sums in the common frame
    if (fl & TDS_LF_PARENT_ADJ) {
      cA = Ia; cP = pa; cC = Ic;
      if constexpr (COR || DER) { cor_cD = cor_D; cor_cH = cor_h; }
      if constexpr (DER) der_cF = der_F;
    } else {
      const int slot = (p >= 0) ? M.acc_slot[p] : M.base_acc;
      if (slot >= 0) {
        if constexpr (!MASS && !CEN && !COR && !DER) acc_add27<RA>(A.ptr<RA>(M.x_acc + slot * M.x_acc_words), ST, Ia, pa);
        rbi_acc<RC>(A.ptr<RC>(M.x_acc + slot * M.x_acc_words + M.x_acc_ic_word), ST, Ic);
        if constexpr (COR || DER) {
          RC* pc = A.ptr<RC>(M.x_acc + slot * M.x_acc_words);
          rbi_acc<RC>(pc, ST, cor_D);
          st6<RC>(pc + 10 * ST, ST, ld6<RC>(pc + 10 * ST, ST) + cor_h);
          if constexpr (DER) st6<RC>(pc + 16 * ST, ST, ld6<RC>(pc + 16 * ST, ST) + der_F);
        }
      }
    }
  }
  if constexpr (DER) {
    if (M.floating) {   // the base's own block from the whole tree's composites, the base body's included (in world axes about O)
      Rbi<RC> Ib = model_rbi_of<RC>(M.base_rbi);
      if constexpr (PAR) { if (pm.any_base) installed_base(Ib); }
      Rbi<RC> Ic; Ic.m = Ib.m; Ic.h = mul(Rb, Ib.h); Ic.I = rot_sym(Rb, Ib.I);
      Rbi<RC> D = cor_rate(Ic, v_base);
      Sv<RC> h = rbi_mul(Ic, v_base);
      if (n_links > 0 && M.parent[0] < 0) { rbi_add(Ic, cC); rbi_add(D, cor_cD); h = h + cor_cH; }
      if (M.base_acc >= 0) {
        const RC* pc = A.ptr<RC>(M.x_acc + M.base_acc * M.x_acc_words);
        rbi_add(Ic, ld_rbi<RC>(A.ptr<RC>(M.x_acc + M.base_acc * M.x_acc_words + M.x_acc_ic_word), ST));
        rbi_add(D, ld_rbi<RC>(pc, ST));
        h = h + ld6<RC>(pc + 10 * ST, ST);
      }
      for (int k = 0; k < 6; ++k) {   // alpha = 0: the twist columns do not move the world
        Sv<RC> S, al, ga, ps;
        der_col(-1, k, S, al, ga, ps);
        const Sv<RC> Fn = rbi_mul(Ic, ga), Fd = rbi_mul(Ic, ps) + rbi_mul(D, S) + cross_mf(S, h);
        const V3<RC> nt = mulT(Rb, Fn.top), nb_ = mulT(Rb, Fn.bot), dt = mulT(Rb, Fd.top), db = mulT(Rb, Fd.bot);
        der_put(0, k, nt.x); der_put(0, n + k, nt.y); der_put(0, 2 * n + k, nt.z);
        der_put(0, 3 * n + k, nb_.x); der_put(0, 4 * n + k, nb_.y); der_put(0, 5 * n + k, nb_.z);
        der_put(1, k, dt.x); der_put(1, n + k, dt.y); der_put(1, 2 * n + k, dt.z);
        der_put(1, 3 * n + k, db.x); der_put(1, 4 * n + k, db.y); der_put(1, 5 * n + k, db.z);
      }
    }
    return;
  }
  if constexpr (COR) {
    if (M.floating) {   // the base's own block from the whole tree's composites, the base body's included (in world axes about O)
      Rbi<RC> Ib = model_rbi_of<RC>(M.base_rbi);
      if constexpr (PAR) { if (pm.any_base) installed_base(Ib); }
      Rbi<RC> Ic; Ic.m = Ib.m; Ic.h = mul(Rb, Ib.h); Ic.I = rot_sym(Rb, Ib.I);
      Rbi<RC> D = cor_rate(Ic, v_base);
      Sv<RC> h = rbi_mul(Ic, v_base);
      if (n_links > 0 && M.parent[0] < 0) { rbi_add(Ic, cC); rbi_add(D, cor_cD); h = h + cor_cH; }
      if (M.base_acc >= 0) {
        const RC* pc = A.ptr<RC>(M.x_acc + M.base_acc * M.x_acc_words);
        rbi_add(Ic, ld_rbi<RC>(A.ptr<RC>(M.x_acc + M.base_acc * M.x_acc_words + M.x_acc_ic_word), ST));
        rbi_add(D, ld_rbi<RC>(pc, ST));
        h = h + ld6<RC>(pc + 10 * ST, ST);
      }
      const Sv<RC> z = Sv<RC>{v3<RC>(RC(0), RC(0), RC(0)), v3<RC>(RC(0), RC(0), RC(0))};
      for (int k = 0; k < 6; ++k) {
        const V3<RC> u = k % 3 == 0 ? col_x(Rb) : (k % 3 == 1 ? col_y(Rb) : col_z(Rb));
        Sv<RC> S = z;
        if (k < 3) S.top = u; else S.bot = u;
        const Sv<RC> F = rbi_mul(Ic, cross_mm(v_base, S)) + cor_B(D, h, S, false);
        const V3<RC> ft = mulT(Rb, F.top), fb = mulT(Rb, F.bot);
        cor_put(k, ft.x); cor_put(n + k, ft.y); cor_put(2 * n + k, ft.z);
        cor_put(3 * n + k, fb.x); cor_put(4 * n + k, fb.y); cor_put(5 * n + k, fb.z);
      }
    }
    return;
  }
  if constexpr (CEN) {
    if (M.floating) {   // the base twist's unit columns [R_b e_k; 0], [0; R_b e_k] move every body: the momentum is the total inertia's
      const Sv<RC> z = Sv<RC>{v3<RC>(RC(0), RC(0), RC(0)), v3<RC>(RC(0), RC(0), RC(0))};
      for (int k = 0; k < 3; ++k) {
        const V3<RC> u = k == 0 ? col_x(Rb) : (k == 1 ? col_y(Rb) : col_z(Rb));
        Sv<RC> s = z; s.top = u; cen_col(k, rbi_mul(cen_I, s));
        s = z; s.bot = u; cen_col(3 + k, rbi_mul(cen_I, s));
      }
    }
    // m, c + O, and the inertia about c: I_O - m (|c|^2 1 - c c^T)
    const RC m = cen_I.m;
    const V3<RC> c = cen_c;
    const RC cc = dot(c, c);
    cen_put(pm.com, 0, m);
    cen_put(pm.com, 1, c.x + O.x); cen_put(pm.com, 2, c.y + O.y); cen_put(pm.com, 3, c.z + O.z);
    cen_put(pm.com, 4, cen_I.I.xx - m * (cc - c.x * c.x)); cen_put(pm.com, 5, cen_I.I.xy + m * c.x * c.y);
    cen_put(pm.com, 6, cen_I.I.xz + m * c.x * c.z); cen_put(pm.com, 7, cen_I.I.yy - m * (cc - c.y * c.y));
    cen_put(pm.com, 8, cen_I.I.yz + m * c.y * c.z); cen_put(pm.com, 9, cen_I.I.zz - m * (cc - c.z * c.z));
    // the bias about c: d/dt k_G = d/dt k_O - (c - O) x d/dt l (the term c' x l vanishes: l = m c')
    const V3<RC> kb = cen_f.top - cross(c, cen_f.bot);
    cen_put(pm.bias, 0, kb.x); cen_put(pm.bias, 1, kb.y); cen_put(pm.bias, 2, kb.z);
    cen_put(pm.bias, 3, cen_f.bot.x); cen_put(pm.bias, 4, cen_f.bot.y); cen_put(pm.bias, 5, cen_f.bot.z);
    return;
  }
  TDSW_PHASE();  // 3

  // ---- base acceleration (forward_dynamics.hpp:218-243) ----------------------------------------------------
  Sv<RA> a_prev;
  Sv<RC> base_acc_b;   // base-frame value of the reference (floating) - needed for qdd[0:6]
  base_acc_b.top = v3<RC>(RC(0), RC(0), RC(0)); base_acc_b.bot = base_acc_b.top;
  if (M.floating) {
    // children sums in the common frame -> base frame (pure rotation: O is the base origin)
    Abi<RA> Ach; Sv<RA> pch; Rbi<RC> Icch;
    Ach.I = {RA(0), RA(0), RA(0), RA(0), RA(0), RA(0)}; Ach.M = Ach.I;
    Ach.H.xx = Ach.H.xy = Ach.H.xz = Ach.H.yx = Ach.H.yy = Ach.H.yz = Ach.H.zx = Ach.H.zy = Ach.H.zz = RA(0);
    pch.top = v3<RA>(RA(0), RA(0), RA(0)); pch.bot = pch.top;
    Icch.m = RC(0); Icch.h = v3<RC>(RC(0), RC(0), RC(0)); Icch.I = {RC(0), RC(0), RC(0), RC(0), RC(0), RC(0)};
    if (n_links > 0 && M.parent[0] < 0) { abi_add(Ach, cA); pch = pch + cP; rbi_add(Icch, cC); }
    if (M.base_acc >= 0) {
      Abi<RA> sa; Sv<RA> sp;
      acc_ld27<RA>(A.ptr<RA>(M.x_acc + M.base_acc * M.x_acc_words), ST, sa, sp);
      abi_add(Ach, sa); pch = pch + sp;
      rbi_add(Icch, ld_rbi<RC>(A.ptr<RC>(M.x_acc + M.base_acc * M.x_acc_words + M.x_acc_ic_word), ST));
    }
    // installed base quantities: (m, h, I about the origin) packed per lane as tds_rbi_pack does on the host, and I_com of the
    // gyroscopic term at fp32 as DevModel::base_inertia_com
    bool base_par = false;
    Rbi<RP> bp;
    if constexpr (PAR) {
      if (pm.any_base) {
        base_par = true;
        RP b[10];
        for (int c = 0; c < 10; ++c) b[c] = par_of(body_slot(0, c), M.base_rbic[c]);
        const RP cc = b[1] * b[1] + b[2] * b[2] + b[3] * b[3];
        bp.m = b[0];
        bp.h = v3<RP>(b[0] * b[1], b[0] * b[2], b[0] * b[3]);
        bp.I.xx = b[4] + b[0] * (cc - b[1] * b[1]);
        bp.I.xy = b[5] - b[0] * b[1] * b[2];
        bp.I.xz = b[6] - b[0] * b[1] * b[3];
        bp.I.yy = b[7] + b[0] * (cc - b[2] * b[2]);
        bp.I.yz = b[8] - b[0] * b[2] * b[3];
        bp.I.zz = b[9] + b[0] * (cc - b[3] * b[3]);
      }
    }
    const M3<RA> Rt = cvt<RA>(transpose(Rb));
    Abi<RA> Ab;
    if constexpr (!MASS) {
      Rbi<RA> rbb = base_par ? cvt_rbi<RA>(bp) : model_rbi_of<RA>(M.base_rbi);
      Ab = abi_from_rbi(rbb);
      Abi<RA> Arot;
      Arot.I = rot_sym(Rt, Ach.I); Arot.M = rot_sym(Rt, Ach.M); Arot.H = rot_gen(Rt, Ach.H);
      abi_add(Ab, Arot);
    }
    Sv<RA> pb;
    if constexpr (!MASS) {
      // gyroscopic bias, kinematics.hpp:54-61 (reference mixes frames here; reproduced as written)
      const M3<RA> RbA = cvt<RA>(Rb);
      M3<RA> Ic0;
      Ic0.xx = RA(M.base_inertia_com[0]); Ic0.xy = RA(M.base_inertia_com[1]); Ic0.xz = RA(M.base_inertia_com[2]);
      Ic0.yx = RA(M.base_inertia_com[3]); Ic0.yy = RA(M.base_inertia_com[4]); Ic0.yz = RA(M.base_inertia_com[5]);
      Ic0.zx = RA(M.base_inertia_com[6]); Ic0.zy = RA(M.base_inertia_com[7]); Ic0.zz = RA(M.base_inertia_com[8]);
      if constexpr (PAR) {
        if (base_par) {
          auto f = [&](int c) -> RA { return RA(f32_round(par_of(body_slot(0, c), M.base_rbic[c]))); };
          Ic0.xx = f(4); Ic0.xy = Ic0.yx = f(5); Ic0.xz = Ic0.zx = f(6); Ic0.yy = f(7); Ic0.yz = Ic0.zy = f(8); Ic0.zz = f(9);
        }
      }
      const M3<RA> Iw = rot_gen(RbA, Ic0);
      const V3<RA> wb = v3<RA>(RA(qdv[0]), RA(qdv[ST]), RA(qdv[2 * ST]));
      pb.top = cross(wb, mul(Iw, wb)) + mul(Rt, pch.top);
      pb.bot = mul(Rt, pch.bot);
      if constexpr (EXT) {   // - f_ext of the base's points in the base frame (O is the base origin)
        const Sv<RC> w = ext_sum(-1, Rb, v3<RC>(RC(0), RC(0), RC(0)));
        pb.top = pb.top - cvt<RA>(mulT(Rb, w.top));
        pb.bot = pb.bot - cvt<RA>(mulT(Rb, w.bot));
      }
    }
    if (any_contact) {  // mass_matrix.hpp:114-120: base block = composite inertia in the base frame
      Rbi<RC> Ib = base_par ? cvt_rbi<RC>(bp) : model_rbi_of<RC>(M.base_rbi);
      const M3<RC> RtC = transpose(Rb);
      Rbi<RC> rot; rot.m = Icch.m; rot.h = mul(RtC, Icch.h); rot.I = rot_sym(RtC, Icch.I);
      rbi_add(Ib, rot);
      const RS z = RS(0);
      RS* b00 = Mb + btri(0, 0) * ST; RS* b10 = Mb + btri(1, 0) * ST; RS* b11 = Mb + btri(1, 1) * ST;
      b00[0] = RS(Ib.I.xx); b00[3 * ST] = RS(Ib.I.xy); b00[4 * ST] = RS(Ib.I.yy); b00[6 * ST] = RS(Ib.I.xz); b00[7 * ST] = RS(Ib.I.yz); b00[8 * ST] = RS(Ib.I.zz);
      // rows 3..5, cols 0..2: H^T with H = h x
      b10[0] = z;               b10[ST] = RS(Ib.h.z);      b10[2 * ST] = RS(-Ib.h.y);
      b10[3 * ST] = RS(-Ib.h.z); b10[4 * ST] = z;           b10[5 * ST] = RS(Ib.h.x);
      b10[6 * ST] = RS(Ib.h.y);  b10[7 * ST] = RS(-Ib.h.x); b10[8 * ST] = z;
      b11[0] = RS(Ib.m); b11[3 * ST] = z; b11[4 * ST] = RS(Ib.m); b11[6 * ST] = z; b11[7 * ST] = z; b11[8 * ST] = RS(Ib.m);
    }
    // -base_abi.inv_mul(bias) with the reference's block inverse (C = -H), inertia.hpp:302-328
    if constexpr (!MASS) {
      M3<RC> I3, H3, M3m;
      I3.xx = Ab.I.xx; I3.xy = Ab.I.xy; I3.xz = Ab.I.xz; I3.yx = Ab.I.xy; I3.yy = Ab.I.yy; I3.yz = Ab.I.yz; I3.zx = Ab.I.xz; I3.zy = Ab.I.yz; I3.zz = Ab.I.zz;
      H3 = cvt<RC>(Ab.H);
      M3m.xx = Ab.M.xx; M3m.xy = Ab.M.xy; M3m.xz = Ab.M.xz; M3m.yx = Ab.M.xy; M3m.yy = Ab.M.yy; M3m.yz = Ab.M.yz; M3m.zx = Ab.M.xz; M3m.zy = Ab.M.yz; M3m.zz = Ab.M.zz;
      auto inv3 = [](const M3<RC>& m) {
        M3<RC> o;
        RC c0 = m.yy * m.zz - m.yz * m.zy, c1 = m.yz * m.zx - m.yx * m.zz, c2 = m.yx * m.zy - m.yy * m.zx;
        RC s = RC(1) / (m.xx * c0 + m.xy * c1 + m.xz * c2);
        o.xx = c0 * s; o.xy = (m.xz * m.zy - m.xy * m.zz) * s; o.xz = (m.xy * m.yz - m.xz * m.yy) * s;
        o.yx = c1 * s; o.yy = (m.xx * m.zz - m.xz * m.zx) * s; o.yz = (m.xz * m.yx - m.xx * m.yz) * s;
        o.zx = c2 * s; o.zy = (m.xy * m.zx - m.xx * m.zy) * s; o.zz = (m.xx * m.yy - m.xy * m.yx) * s;
        return o;
      };
      auto neg = [](M3<RC> m) { m.xx = -m.xx; m.xy = -m.xy; m.xz = -m.xz; m.yx = -m.yx; m.yy = -m.yy; m.yz = -m.yz; m.zx = -m.zx; m.zy = -m.zy; m.zz = -m.zz; return m; };
      auto sub = [](M3<RC> a, const M3<RC>& b) { a.xx -= b.xx; a.xy -= b.xy; a.xz -= b.xz; a.yx -= b.yx; a.yy -= b.yy; a.yz -= b.yz; a.zx -= b.zx; a.zy -= b.zy; a.zz -= b.zz; return a; };
      auto add = [](M3<RC> a, const M3<RC>& b) { a.xx += b.xx; a.xy += b.xy; a.xz += b.xz; a.yx += b.yx; a.yy += b.yy; a.yz += b.yz; a.zx += b.zx; a.zy += b.zy; a.zz += b.zz; return a; };
      M3<RC> Ainv = inv3(I3);
      M3<RC> C = neg(H3);
      M3<RC> D = inv3(sub(M3m, mul(mul(C, Ainv), H3)));
      M3<RC> AinvBD = mul(mul(Ainv, H3), D);
      M3<RC> Ii = add(Ainv, mul(mul(AinvBD, C), Ainv));
      M3<RC> Hi = neg(AinvBD);
      V3<RC> ft = cvt<RC>(pb.top), fb = cvt<RC>(pb.bot);
      V3<RC> at = mul(Ii, ft) + mul(Hi, fb);
      V3<RC> ab = mul(D, fb) + mulT(Hi, ft);
      base_acc_b.top = v3<RC>(-at.x, -at.y, -at.z);
      base_acc_b.bot = v3<RC>(-ab.x, -ab.y, -ab.z);
    }
    a_prev.top = cvt<RA>(mul(Rb, base_acc_b.top));
    a_prev.bot = cvt<RA>(mul(Rb, base_acc_b.bot));
  } else {
    a_prev.top = v3<RA>(RA(0), RA(0), RA(0));
    a_prev.bot = v3<RA>(RA(-P.gravity[0]), RA(-P.gravity[1]), RA(-P.gravity[2]));
  }
  if constexpr (MINV) {
    auto put = [&](int k, RS x) {
      if constexpr (AD) io.jac[((size_t)k * io.jac_n_in + jcol) * ns + e] = x.d;
      else io.jac[(size_t)k * ns + e] = x;
    };
    // blocked Cholesky M = L L^T, the contact solve's loop
    for (int bi = 0; bi < nb; ++bi) {
      for (int bj = 0; bj <= bi; ++bj) {
        B9<RS> Ab = ldb<RS>(Mb + btri(bi, bj) * ST, ST);
        for (int bk = 0; bk < bj; ++bk)
          gemm_nt_sub(Ab, ldb<RS>(Mb + btri(bi, bk) * ST, ST), ldb<RS>(Mb + btri(bj, bk) * ST, ST));
        if (bj < bi) stb<RS>(Mb + btri(bi, bj) * ST, ST, mul_linvT(Ab, ldl6<RS>(dinv + bj * 6 * ST, ST)));
        else stl6<RS>(dinv + bi * 6 * ST, ST, chol3_inv(Ab));
      }
    }
    // W = L^-1: W_ij = -W_ii sum_{j <= k < i} L_ik W_kj.  Column j top down reads L in the columns right of j and W above row i.
    for (int bj = 0; bj < nb; ++bj) {
      const B9<RS> Wjj = l6_full(ldl6<RS>(dinv + bj * 6 * ST, ST));
      for (int bi = bj + 1; bi < nb; ++bi) {
        B9<RS> X = b9_zero<RS>();
        gemm_nn_sub(X, ldb<RS>(Mb + btri(bi, bj) * ST, ST), Wjj);
        for (int bk = bj + 1; bk < bi; ++bk)
          gemm_nn_sub(X, ldb<RS>(Mb + btri(bi, bk) * ST, ST), ldb<RS>(Mb + btri(bk, bj) * ST, ST));
        stb<RS>(Mb + btri(bi, bj) * ST, ST, linv_mul(ldl6<RS>(dinv + bi * 6 * ST, ST), X));
      }
    }
    // M^-1 block (i, j), i >= j: sum_{k >= i} W_ki^T W_kj
    if (live && io.jac) {
      for (int bi = 0; bi < nb; ++bi) {
        const B9<RS> Wii = l6_full(ldl6<RS>(dinv + bi * 6 * ST, ST));
        for (int bj = 0; bj <= bi; ++bj) {
          B9<RS> X = b9_zero<RS>();
          gemm_tn_add(X, Wii, bj == bi ? Wii : ldb<RS>(Mb + btri(bi, bj) * ST, ST));
          for (int bk = bi + 1; bk < nb; ++bk)
            gemm_tn_add(X, ldb<RS>(Mb + btri(bk, bi) * ST, ST), ldb<RS>(Mb + btri(bk, bj) * ST, ST));
          for (int a = 0; a < 3; ++a)
            for (int b = 0; b < 3; ++b) {
              const int r = 3 * bi + a, c = 3 * bj + b;
              if (r >= n || c > r) continue;
              put(r * n + c, X.a[a * 3 + b]);
              if (c < r) put(c * n + r, X.a[a * 3 + b]);
            }
        }
      }
    }
    return;
  }
  if constexpr (MASS) {   // dense symmetric M from the blocked lower triangle (the padding dofs are not written)
    if (live && io.jac) {
      auto put = [&](int k, RS x) {
        if constexpr (AD) io.jac[((size_t)k * io.jac_n_in + jcol) * ns + e] = x.d;
        else io.jac[(size_t)k * ns + e] = x;
      };
      for (int r = 0; r < n; ++r)
        for (int c = 0; c <= r; ++c) {
          const RS x = Mb[(btri(r / 3, c / 3) + (r % 3) * 3 + (c % 3)) * ST];
          put(r * n + c, x);
          if (c < r) put(c * n + r, x);
        }
    }
    return;
  }
  const Sv<RA> a_base = a_prev;
  const RA dtA = RA(P.dt);

  // ---- pass 3: root -> leaf (forward_dynamics.hpp:245-302) + integrate_euler_qdd (integrator.hpp:141-195) ----
  for (int i = 0; i < n_links; ++i) {
    const int p = M.parent[i];
    const int fl = M.flags[i];
    RA* const vrec = A.ptr<RA>(M.x_link + i * LWD + VOFF);
    Sv<RA> a;
    if (fl & TDS_LF_PARENT_ADJ) a = a_prev;
    else if (p >= 0) a = ld6<RA>(A.ptr<RA>(M.x_link + p * LWD + VOFF), ST);
    else a = a_base;
    if (fl & TDS_LF_SPHERICAL) {   // forward_dynamics.hpp:272-284: qdd = D^-1 (u - U^T a)
      const RA* urec = A.ptr<RA>(M.x_link + i * LWD);
      const int d0 = M.qd_idx[i];
      a = a + ld6<RA>(vrec, ST);
      RA t[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) t[k] = urec[(27 + k) * ST] - dot(ld6<RA>(urec + k * 6 * ST, ST), a);
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        const RA qdd = urec[(18 + j * 3) * ST] * t[0] + urec[(18 + j * 3 + 1) * ST] * t[1] + urec[(18 + j * 3 + 2) * ST] * t[2];
        const Sv<RA> S = cvt_sv<RA>(S_col(i, j));
        a.top = axpy(S.top, qdd, a.top);
        a.bot = axpy(S.bot, qdd, a.bot);
        if (mode == MODE_FD) {
          if constexpr (AD) { if (live && io.jac) io.jac[((size_t)(d0 + j) * io.jac_n_in + jcol) * ns + e] = qdd.d; }
          else if constexpr (TP) qdv[(d0 + j) * ST] = qdd;   // the VJP's output rows (qd is not read again in this mode)
          else if (live && io.qdd_out) io.qdd_out[(size_t)(d0 + j) * ns + e] = (float)val_of(qdd);
        } else if (!world_step) qdv[(d0 + j) * ST] = RQ(RA(qdv[(d0 + j) * ST]) + qdd * dtA);
      }
    } else if (!(fl & TDS_LF_FIXED)) {
      const RA* urec = A.ptr<RA>(M.x_link + i * LWD);
      const Sv<RA> c = ld6<RA>(vrec, ST);
      const Sv<RA> U = ld6<RA>(urec, ST);
      a = a + c;
      const RA qdd = urec[6 * ST] * (urec[7 * ST] - dot(U, a));
      const Sv<RA> S = cvt_sv<RA>(ld6<RC>(Sw + i * 6 * ST, ST));
      a.top = axpy(S.top, qdd, a.top);
      a.bot = axpy(S.bot, qdd, a.bot);
      const int qdi = M.qd_idx[i];
      if (mode == MODE_FD) {
        if constexpr (AD) { if (live && io.jac) io.jac[((size_t)qdi * io.jac_n_in + jcol) * ns + e] = qdd.d; }
        else if constexpr (TP) qdv[qdi * ST] = qdd;
        else if (live && io.qdd_out) io.qdd_out[(size_t)qdi * ns + e] = (float)val_of(qdd);
      } else if (!world_step) qdv[qdi * ST] = RQ(RA(qdv[qdi * ST]) + qdd * dtA);
    }
    st6<RA>(vrec, ST, a);
    a_prev = a;
  }
  if (M.floating) {  // forward_dynamics.hpp:317-322 (gravity added un-rotated), integrator.hpp:153-163
    const RC qb[6] = {base_acc_b.top.x, base_acc_b.top.y, base_acc_b.top.z, base_acc_b.bot.x + RC(P.gravity[0]),
                      base_acc_b.bot.y + RC(P.gravity[1]), base_acc_b.bot.z + RC(P.gravity[2])};
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      if (mode == MODE_FD) {
        if constexpr (AD) { if (live && io.jac) io.jac[((size_t)k * io.jac_n_in + jcol) * ns + e] = qb[k].d; }
        else if constexpr (TP) qdv[k * ST] = qb[k];
        else if (live && io.qdd_out) io.qdd_out[(size_t)k * ns + e] = (float)val_of(qb[k]);
      } else if (!world_step) qdv[k * ST] = RQ(RC(qdv[k * ST]) + qb[k] * RC(P.dt));
    }
  }
  TDSW_PHASE();  // 4
  if constexpr (TP) { if (mode == MODE_FD) { vjp_write(n, [&](int r) { return qdv[r * ST].id; }); return; } }
  if (mode == MODE_FD) return;

  // ---- contact solve -------------------------------------------------------------------------------------------
  __syncwarp();   // the Y rows below reuse the per-link records with another lane interleave
  if ((mode == MODE_FULL || world_step) && any_contact) {
    // blocked Cholesky M = L L^T (3x3 blocks, lower): off-diagonal blocks of L overwrite M, diagonal blocks are
    // kept as their inverses.  (The reference inverts M, tiny_matrix_x.h:240-344; only M^-1 products are needed.)
    for (int bi = 0; bi < nb; ++bi) {
      for (int bj = 0; bj <= bi; ++bj) {
        B9<RS> Ab = ldb<RS>(Mb + btri(bi, bj) * ST, ST);
        for (int bk = 0; bk < bj; ++bk)
          gemm_nt_sub(Ab, ldb<RS>(Mb + btri(bi, bk) * ST, ST), ldb<RS>(Mb + btri(bj, bk) * ST, ST));
        if (bj < bi) stb<RS>(Mb + btri(bi, bj) * ST, ST, mul_linvT(Ab, ldl6<RS>(dinv + bj * 6 * ST, ST)));
        else stl6<RS>(dinv + bi * 6 * ST, ST, chol3_inv(Ab));
      }
    }
    TDSW_PHASE();  // 5
    const V3<RC> nbv = v3<RC>(-pn.x, -pn.y, -pn.z);                     // world_normal_on_b of every plane contact
    const V3<RC> f1 = v3<RC>(RC(M.fr1[0]), RC(M.fr1[1]), RC(M.fr1[2]));
    const V3<RC> f2 = v3<RC>(RC(M.fr2[0]), RC(M.fr2[1]), RC(M.fr2[2]));
    // One LCP per list of World::mb_contacts_, solved one after the other, each from the velocities the previous one left
    // (world.hpp:351-355).  Group 0: every plane contact (the plane is multibody 0; its lists (plane, b) share no dof, so
    // their Gauss-Seidel sweeps do not see each other and one LCP over all of them is the same arithmetic).  Groups 1..: the
    // pairs of multibodies (a, b) in lexicographic order, rows J_b - J_a over the dofs of both.
    // CF: the impulse rows of active contact c of group grp (pair records at prec): F = -(p0 n_b + p1 t1 + p2 t2) on body b
    auto cf_impulse = [&](int grp, int c, const RC* prec, RS p0, RS p1, RS p2) {
      if constexpr (CF) {
        int k;
        V3<RC> n_b, t1, t2;
        if (grp == 0) { k = cf_nth_bit(cf_plane, c); n_b = nbv; t1 = f1; t2 = f2; }
        else {
          const int lo = M.pg_begin[grp - 1];
          k = pt_index + lo + cf_nth_bit(cf_pair >> lo, c);
          n_b = ld3<RC>(prec + (c * 9 + 3) * ST, ST);
          plane_space_t(n_b, t1, t2);
        }
        const V3<RC> F = n_b * RC(p0) + t1 * RC(p1) + t2 * RC(p2);
        cf_put(10 * k + 7, -F.x); cf_put(10 * k + 8, -F.y); cf_put(10 * k + 9, -F.z);
      }
    };
    int pbase = 0;   // first record of the current pair group
    for (int grp = 0; grp <= M.n_pair_groups; ++grp) {
    const int n_act = grp == 0 ? n_active : pgc[grp - 1];
    const RC* const prec = A.ptr<RC>(M.x_pcon + pbase * 9 * RCW);       // records of this pair group
    if (grp > 0) pbase += n_act;
    const int max_active = __reduce_max_sync(0xffffffffu, n_act);
    if (max_active == 0) {
      if (grp == 0) { TDSW_PHASE(); TDSW_PHASE(); }
      continue;
    }
    for (int c = 0; c < max_active; ++c) {
      if (c < n_act) {
        if (grp == 0) {
          const RC* pc = A.ptr<RC>(M.x_con + c * 5 * RCW);
          RS* const Y = A.ptr<RS>(M.x_Y) + c * n3 * 3 * ST;       // [dof k][rhs] : element (3k + rhs)
          const V3<RC> xc = ld3<RC>(pc, ST);
          const RC dist = pc[3 * ST];
          const int L = (int)val_of(pc[4 * ST]);
          for (int k = 0; k < 3 * n3; ++k) Y[k * ST] = RS(0);
          V3<RC> vel = v3<RC>(RC(0), RC(0), RC(0));                  // vel_b = J qd
          if (M.floating) {  // jacobian.hpp:39-58 with r = x_c (O is the base origin)
            const V3<RC> cols[6] = {v3<RC>(RC(0), -xc.z, xc.y), v3<RC>(xc.z, RC(0), -xc.x), v3<RC>(-xc.y, xc.x, RC(0)),
                                    v3<RC>(RC(1), RC(0), RC(0)), v3<RC>(RC(0), RC(1), RC(0)), v3<RC>(RC(0), RC(0), RC(1))};
  #pragma unroll
            for (int k = 0; k < 6; ++k) {
              Y[(3 * k) * ST] = RS(dot(nbv, cols[k])); Y[(3 * k + 1) * ST] = RS(dot(f1, cols[k])); Y[(3 * k + 2) * ST] = RS(dot(f2, cols[k]));
              vel = vel + cols[k] * RC(qdv[k * ST]);
            }
          }
          for (int j = L; j >= 0; j = M.parent[j]) {  // jacobian.hpp:63-80: column = S_j evaluated at the contact point
            const int nc = n_cols(j);
            for (int cj = 0; cj < nc; ++cj) {
              const Sv<RC> S = S_col(j, cj);
              const V3<RC> col = S.bot + cross(S.top, xc);
              const int qj = M.qd_idx[j] + cj;
              Y[(3 * qj) * ST] = RS(dot(nbv, col)); Y[(3 * qj + 1) * ST] = RS(dot(f1, col)); Y[(3 * qj + 2) * ST] = RS(dot(f2, col));
              vel = vel + col * RC(qdv[qj * ST]);
            }
          }
          // rel_vel = vel_a - vel_b = -vel ; mb_constraint_solver.hpp:299-345
          RS* const cs = A.ptr<RS>(M.x_conS) + c * 6 * ST;   // b[3], x[3]
          if (P.contact_model == 1) cs[0] = RS(dot(nbv, vel));   // spring-damper: approach speed n_b . v_b
          else cs[0] = RS((RC(1) + RC(par_of(par_restitution, P.restitution))) * dot(nbv, vel) - RC(P.erp) * dist / RC(P.dt));
          cs[ST] = RS(dot(f1, vel));
          cs[2 * ST] = RS(dot(f2, vel));
          cs[3 * ST] = RS(0); cs[4 * ST] = RS(0); cs[5 * ST] = RS(0);
        } else {
          // a contact between two multibodies: point on a / on b at the links la / lb, normal on b, friction directions of
          // plane_space(normal) (mb_constraint_solver.hpp:359-363, 506-520)
          const RC* pc = prec + c * 9 * ST;
          RS* const Y = A.ptr<RS>(M.x_Y) + c * n3 * 3 * ST;
          const V3<RC> xa = ld3<RC>(pc, ST), nrm = ld3<RC>(pc + 3 * ST, ST);
          const RC dist = pc[6 * ST];
          const int la = (int)val_of(pc[7 * ST]), lb = (int)val_of(pc[8 * ST]);
          const V3<RC> xb = xa - nrm * dist;
          V3<RC> g1, g2;
          plane_space_t(nrm, g1, g2);
          for (int k = 0; k < 3 * n3; ++k) Y[k * ST] = RS(0);
          V3<RC> vel = v3<RC>(RC(0), RC(0), RC(0));                  // vel_b - vel_a = -rel_vel
          for (int j = lb; j >= 0; j = M.parent[j]) {
            const int nc = n_cols(j);
            for (int cj = 0; cj < nc; ++cj) {
              const Sv<RC> S = S_col(j, cj);
              const V3<RC> col = S.bot + cross(S.top, xb);
              const int qj = M.qd_idx[j] + cj;
              Y[(3 * qj) * ST] = RS(dot(nrm, col)); Y[(3 * qj + 1) * ST] = RS(dot(g1, col)); Y[(3 * qj + 2) * ST] = RS(dot(g2, col));
              vel = vel + col * RC(qdv[qj * ST]);
            }
          }
          for (int j = la; j >= 0; j = M.parent[j]) {
            const int nc = n_cols(j);
            for (int cj = 0; cj < nc; ++cj) {
              const Sv<RC> S = S_col(j, cj);
              const V3<RC> col = S.bot + cross(S.top, xa);
              const int qj = M.qd_idx[j] + cj;
              Y[(3 * qj) * ST] = RS(-dot(nrm, col)); Y[(3 * qj + 1) * ST] = RS(-dot(g1, col)); Y[(3 * qj + 2) * ST] = RS(-dot(g2, col));
              vel = vel - col * RC(qdv[qj * ST]);
            }
          }
          RS* const cs = A.ptr<RS>(M.x_conS) + c * 6 * ST;   // b[3], x[3]
          if (P.contact_model == 1) cs[0] = RS(dot(nrm, vel));
          else cs[0] = RS((RC(1) + RC(par_of(par_restitution, P.restitution))) * dot(nrm, vel) - RC(P.erp) * dist / RC(P.dt));
          cs[ST] = RS(dot(g1, vel));
          cs[2 * ST] = RS(dot(g2, vel));
          cs[3 * ST] = RS(0); cs[4 * ST] = RS(0); cs[5 * ST] = RS(0);
        }
        RS* const Y = A.ptr<RS>(M.x_Y) + c * n3 * 3 * ST;
        // Y <- L^-1 Y (blocked forward substitution, 3 right-hand sides)
        for (int bi = 0; bi < nb; ++bi) {
          B9<RS> a = ldb<RS>(Y + bi * 9 * ST, ST);
          for (int bk = 0; bk < bi; ++bk) gemm_nn_sub(a, ldb<RS>(Mb + btri(bi, bk) * ST, ST), ldb<RS>(Y + bk * 9 * ST, ST));
          stb<RS>(Y + bi * 9 * ST, ST, linv_mul(ldl6<RS>(dinv + bi * 6 * ST, ST), a));
        }
      }
    }
    if (grp == 0) TDSW_PHASE();  // 6
    // matrix-free projected Gauss-Seidel on w = Y p; row order normals | friction-1 | friction-2
    // (solve_pgs, mb_constraint_solver.hpp:101-142; bounds :417-436)
    for (int k = 0; k < n3; ++k) wv[k * ST] = RS(0);
    const RS cfm = RS(P.cfm), mu = RS(par_of(par_friction, P.friction));
    if (P.contact_model == 1) {
      // Spring-damper law instead of the LCP (DESIGN.md "Spring-damper contacts"; parity unpinned): closed-form impulses
      //   p_n = dt max(0, k x^n + d x^n xdot),  x = -distance, xdot = n_b . v_b
      //   p_t = dt mu f_n tanh(|v_t| / v_transition) v_t / |v_t|   along the two friction directions
      // accumulated into w = Y p like the Gauss-Seidel impulses; the back substitution below is shared.
      for (int c = 0; c < max_active; ++c) {
        if (c < n_act) {
          const RS* cs = A.ptr<RS>(M.x_conS) + c * 6 * ST;
          const RS x = RS(-(grp == 0 ? A.ptr<RC>(M.x_con + c * 5 * RCW)[3 * ST] : prec[(c * 9 + 6) * ST]));
          const RS vn = cs[0], v1 = cs[ST], v2 = cs[2 * ST];
          const RS xn = pow_t(x, RS(P.exponent_n));
          RS fn = RS(P.spring_k) * xn + RS(P.damper_d) * xn * vn;
          if (P.hard_contact_condition && fn < RS(0)) fn = RS(0);
          const RS vt = sqrt_t(v1 * v1 + v2 * v2);
          const RS sc = vt > RS(1e-12) ? mu * fn * tanh_t(vt / RS(P.v_transition)) / vt * RS(P.dt) : RS(0);
          const RS p[3] = {fn * RS(P.dt), sc * v1, sc * v2};
          if constexpr (CF) cf_impulse(grp, c, prec, p[0], p[1], p[2]);
          const RS* y = A.ptr<RS>(M.x_Y) + (c * n3 * 3) * ST;
          for (int k = 0; k < n3; ++k)
            wv[k * ST] += p[0] * y[(3 * k) * ST] + p[1] * y[(3 * k + 1) * ST] + p[2] * y[(3 * k + 2) * ST];
        }
      }
    } else
    for (int it = 0; it < P.pgs_iterations; ++it) {
      for (int blk = 0; blk < 3; ++blk) {
        for (int c = 0; c < max_active; ++c) {
          if (c < n_act) {
            RS* const cs = A.ptr<RS>(M.x_conS) + c * 6 * ST;
            const RS* y = A.ptr<RS>(M.x_Y) + (c * n3 * 3 + blk) * ST;     // element k at y[3k * ST]
            RS yy0 = RS(0), yy1 = RS(0), yy2 = RS(0), yw0 = RS(0), yw1 = RS(0), yw2 = RS(0);
            for (int b = 0; b < nb; ++b) {
              const RS y0 = y[(9 * b) * ST], y1 = y[(9 * b + 3) * ST], y2 = y[(9 * b + 6) * ST];
              yy0 += y0 * y0; yy1 += y1 * y1; yy2 += y2 * y2;
              yw0 += y0 * wv[(3 * b) * ST]; yw1 += y1 * wv[(3 * b + 1) * ST]; yw2 += y2 * wv[(3 * b + 2) * ST];
            }
            const RS yy = (yy0 + yy1) + yy2, yw = (yw0 + yw1) + yw2;
            const RS x_old = cs[(3 + blk) * ST];
            RS x = (cs[blk * ST] - yw + yy * x_old) / (yy + cfm);
            if (blk == 0) {
              x = x < RS(0) ? RS(0) : x;
              x = x > RS(100000) ? RS(100000) : x;
            } else {
              RS s = cs[3 * ST];
              s = s < RS(0) ? RS(0) : s;
              const RS lim = mu * s;
              x = x < -lim ? -lim : x;
              x = x > lim ? lim : x;
            }
            cs[(3 + blk) * ST] = x;
            const RS dx = x - x_old;
            for (int b = 0; b < nb; ++b) {
              wv[(3 * b) * ST] += dx * y[(9 * b) * ST];
              wv[(3 * b + 1) * ST] += dx * y[(9 * b + 3) * ST];
              wv[(3 * b + 2) * ST] += dx * y[(9 * b + 6) * ST];
            }
          }
        }
      }
    }
    if constexpr (CF) {
      if (P.contact_model != 1)
        for (int c = 0; c < n_act; ++c) {
          const RS* cs = A.ptr<RS>(M.x_conS) + c * 6 * ST;
          cf_impulse(grp, c, prec, cs[3 * ST], cs[4 * ST], cs[5 * ST]);
        }
    }
    if (grp == 0) TDSW_PHASE();  // 7
    // qd_b -= M^-1 Jc^T p = L^-T w   (mb_constraint_solver.hpp:476-497), blocked back substitution
    for (int bi = nb - 1; bi >= 0; --bi) {
      RS a0 = wv[(3 * bi) * ST], a1 = wv[(3 * bi + 1) * ST], a2 = wv[(3 * bi + 2) * ST];
      for (int bk = bi + 1; bk < nb; ++bk) {
        const B9<RS> Lb = ldb<RS>(Mb + btri(bk, bi) * ST, ST);
        const RS z0 = wv[(3 * bk) * ST], z1 = wv[(3 * bk + 1) * ST], z2 = wv[(3 * bk + 2) * ST];
        a0 -= Lb.a[0] * z0 + Lb.a[3] * z1 + Lb.a[6] * z2;
        a1 -= Lb.a[1] * z0 + Lb.a[4] * z1 + Lb.a[7] * z2;
        a2 -= Lb.a[2] * z0 + Lb.a[5] * z1 + Lb.a[8] * z2;
      }
      const L6<RS> li = ldl6<RS>(dinv + bi * 6 * ST, ST);
      const RS z0 = li.i00 * a0 + li.i10 * a1 + li.i20 * a2;
      const RS z1 = li.i11 * a1 + li.i21 * a2;
      const RS z2 = li.i22 * a2;
      wv[(3 * bi) * ST] = z0; wv[(3 * bi + 1) * ST] = z1; wv[(3 * bi + 2) * ST] = z2;
    }
    if (n_act > 0)
      for (int k = 0; k < n; ++k) qdv[k * ST] = RQ(RS(qdv[k * ST]) - wv[k * ST]);
    }   // groups
  }
  TDSW_PHASE();  // 8

  // ---- integrate_euler with qdd = 0 (integrator.hpp:10-133) -----------------------------------------------------
  RC up_z = RC(1);
  if (M.floating && !world_step) {
    const RC h = RC(0.5) * RC(P.dt);
    RC qx = RC(qv[0]), qy = RC(qv[ST]), qz = RC(qv[2 * ST]), qw = RC(qv[3 * ST]);
    const RC w0 = RC(qdv[0]), w1 = RC(qdv[ST]), w2 = RC(qdv[2 * ST]);
    const RC dw = (-qx * w0 - qy * w1 - qz * w2) * h;
    const RC dx = (qw * w0 + qz * w1 - qy * w2) * h;
    const RC dy = (qw * w1 + qx * w2 - qz * w0) * h;
    const RC dz = (qw * w2 + qy * w0 - qx * w1) * h;
    qx += dx; qy += dy; qz += dz; qw += dw;
    const RC len = sqrt_t(qx * qx + qy * qy + qz * qz + qw * qw);
    qx /= len; qy /= len; qz /= len; qw /= len;
    qv[0] = RQ(qx); qv[ST] = RQ(qy); qv[2 * ST] = RQ(qz); qv[3 * ST] = RQ(qw);
    for (int k = 0; k < 3; ++k)
      qv[(4 + k) * ST] = RQ(RC(qv[(4 + k) * ST]) + RC(qdv[(3 + k) * ST]) * RC(P.dt));
    up_z = RC(1) - RC(2) * (qx * qx + qy * qy) / (qx * qx + qy * qy + qz * qz + qw * qw);
  }
  for (int i = 0; i < n_links && !world_step; ++i) {
    if (M.flags[i] & TDS_LF_FIXED) continue;
    if (M.flags[i] & TDS_LF_SPHERICAL) {
      // integrator.hpp:97-122: the joint velocity is damped by MultiBody::joint_damping_ ^ (1000 dt) (default 0.995,
      // multi_body.hpp:51) in every integrate_euler, then q += quat_velocity_spherical(q, qd, dt), normalised
      const int q0 = M.q_idx[i], d0 = M.qd_idx[i];
      const RC damp = RC(pow(0.995, P.dt * 1000.0));
      RC w[3];
      for (int k = 0; k < 3; ++k) { w[k] = RC(qdv[(d0 + k) * ST]) * damp; qdv[(d0 + k) * ST] = RQ(w[k]); }
      const RC h = RC(0.5) * RC(P.dt);
      RC qx = RC(qv[q0 * ST]), qy = RC(qv[(q0 + 1) * ST]), qz = RC(qv[(q0 + 2) * ST]), qw = RC(qv[(q0 + 3) * ST]);
      const RC dw = (-qx * w[0] - qy * w[1] - qz * w[2]) * h;      // tiny_algebra.hpp:616-627
      const RC dx = (qw * w[0] + qy * w[2] - qz * w[1]) * h;
      const RC dy = (qw * w[1] + qz * w[0] - qx * w[2]) * h;
      const RC dz = (qw * w[2] + qx * w[1] - qy * w[0]) * h;
      qx += dx; qy += dy; qz += dz; qw += dw;
      const RC len = sqrt_t(qx * qx + qy * qy + qz * qz + qw * qw);
      qv[q0 * ST] = RQ(qx / len); qv[(q0 + 1) * ST] = RQ(qy / len); qv[(q0 + 2) * ST] = RQ(qz / len); qv[(q0 + 3) * ST] = RQ(qw / len);
      continue;
    }
    const int qi = M.q_idx[i];
    qv[qi * ST] = RQ(RC(qv[qi * ST]) + RC(qdv[M.qd_idx[i] * ST]) * RC(P.dt));
  }

  // ---- reward / done / auto-reset, write back ------------------------------------------------------------------------
  if constexpr (AD) {   // the Jacobian column of this lane's direction: rows q' | qd'
    if (live && io.jac) {
      for (int k = 0; k < M.n_q; ++k) io.jac[((size_t)k * io.jac_n_in + jcol) * ns + e] = qv[k * ST].d;
      for (int k = 0; k < n; ++k) io.jac[((size_t)(M.n_q + k) * io.jac_n_in + jcol) * ns + e] = qdv[k * ST].d;
    }
    return;
  }
  if constexpr (TP) {   // rows q' | qd'
    vjp_write(M.n_q + n, [&](int r) { return r < M.n_q ? qv[r * ST].id : qdv[(r - M.n_q) * ST].id; });
    return;
  }
  if (live) {
    bool done = false;
    if (E.reward_kind == 1) {   // laikago_environment2.h:130-171 (fixed-base emulation)
      const float x = (float)val_of(qv[0]), z = (float)val_of(qv[2 * ST]);
      const float upz = cosf((float)val_of(qv[3 * ST])) * cosf((float)val_of(qv[4 * ST]));
      done = (upz < 0.6f) || (z < 0.2f);
      if (io.reward) io.reward[e] = done ? 0.f : x;
    } else if (E.reward_kind == 2) {
      const float x = (float)val_of(qv[4 * ST]), z = (float)val_of(qv[6 * ST]);
      done = ((float)val_of(up_z) < 0.6f) || (z < 0.2f);
      if (io.reward) io.reward[e] = done ? 0.f : x;
    } else if (E.reward_kind == 3) {   // ant_environment2.h:75-105: done = z < 0.26, reward = (x' - x)/dt, which integrate_euler makes the x velocity
      done = (float)val_of(qv[2 * ST]) < 0.26f;
      if (io.reward) io.reward[e] = done ? 0.f : (float)val_of(qdv[0]);
    }
    if (io.done && E.reward_kind) io.done[e] = done ? 1.f : 0.f;
    if (done && E.auto_reset) {   // ars_vectorized_environment.h:262-283
      for (int k = 0; k < M.n_q; ++k) io.q_out[(size_t)k * ns + e] = E.reset_q[k];
      for (int k = 0; k < n; ++k) io.qd_out[(size_t)k * ns + e] = 0.f;
    } else {
      for (int k = 0; k < M.n_q; ++k) io.q_out[(size_t)k * ns + e] = (float)val_of(qv[k * ST]);
      for (int k = 0; k < n; ++k) io.qd_out[(size_t)k * ns + e] = (float)val_of(qdv[k * ST]);
    }
  }
  TDSW_PHASE();  // 9
}

}  // namespace tdsw

#ifndef TDS_STEPW_KERNEL_ONLY   // (tests/cpp/stepw_host.cpp compiles the kernel above for the host, without the launchers)
extern "C" int tds_launch_stepw(const DevModel* M, const SimParams* P, const EnvParams* E, const StepIO* io,
                                int mode, int use_pd, int precision, char* gscratch, int use_smem,
                                int warps_per_block, cudaStream_t stream) {
  using namespace tdsw;
  const int threads = 32 * warps_per_block;
  const int blocks = (io->n + threads - 1) / threads;
  const size_t smem = use_smem ? (size_t)warps_per_block * M->x_total * 32 * 4 : 0;
  cudaError_t err = cudaSuccess;
#define TDSW_LAUNCH(RA, RC, RS, SM)                                                                     \
  do {                                                                                                  \
    auto k = tds_stepw_kernel<RA, RC, RS, float, SM>;                                                   \
    static size_t smem_set_dev[64] = {0}; int dev_ = 0; cudaGetDevice(&dev_); size_t& smem_set = smem_set_dev[dev_ & 63]; \
    if (smem > 48 * 1024 && smem > smem_set) {                                                          \
      err = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);            \
      if (err == cudaSuccess) smem_set = smem;                                                          \
    }                                                                                                   \
    if (err == cudaSuccess) {                                                                           \
      k<<<blocks, threads, smem, stream>>>(*M, *P, *E, *io, mode, use_pd, gscratch, NoPar{});           \
      err = cudaGetLastError();                                                                         \
    }                                                                                                   \
  } while (0)
  if (precision == 0) { if (use_smem) TDSW_LAUNCH(float, double, float, true); else TDSW_LAUNCH(float, double, float, false); }
  else if (precision == 1) { if (use_smem) TDSW_LAUNCH(double, double, double, true); else TDSW_LAUNCH(double, double, double, false); }
  else { if (use_smem) TDSW_LAUNCH(float, float, float, true); else TDSW_LAUNCH(float, float, float, false); }
#undef TDSW_LAUNCH
  return (int)err;
}

// Differentiable step: the same kernel on forward-mode dual numbers (fp64), one lane per (environment, input direction).
// M must carry the 16-byte layout (tds_build_layout_w(..., 16, 16, 16, -1, 16)); gscratch: n_dirs * ceil(n / 32) blocks of
// x_total * 128 bytes; directions [io->jac_dir0, io->jac_dir0 + n_dirs) are computed by this launch.
extern "C" int tds_launch_stepw_jacobian(const DevModel* M, const SimParams* P, const EnvParams* E, const StepIO* io, int mode,
                                         int use_pd, int n_dirs, char* gscratch, cudaStream_t stream) {
  using namespace tdsw;
  typedef tds::Dual<double> D;
  const dim3 grid((io->n + 31) / 32, n_dirs);
  tds_stepw_kernel<D, D, D, D, false><<<grid, 32, 0, stream>>>(*M, *P, *E, *io, mode, use_pd, gscratch, NoPar{});
  return (int)cudaGetLastError();
}

// Vector-Jacobian product: the same kernel on the taping scalar (fp64), one lane per environment, 32 lanes per block.  M must
// carry the 16-byte layout; gscratch: ceil(n / 32) blocks of x_total * 128 bytes; io->tape / io->tape_adj: ceil(n / 32) * 32
// lanes of io->tape_cap nodes / adjoints; io->g_out -> io->g_in.  *io->tape_overflow is set when a lane's tape was too short
// (its g_in column is then not written).
extern "C" int tds_launch_stepw_vjp(const DevModel* M, const SimParams* P, const EnvParams* E, const StepIO* io, int mode,
                                    int use_pd, char* gscratch, cudaStream_t stream) {
  using namespace tdsw;
  typedef tds::Tape<double> T;
  tds_stepw_kernel<T, T, T, T, false><<<(io->n + 31) / 32, 32, 0, stream>>>(*M, *P, *E, *io, mode, use_pd, gscratch, NoPar{});
  return (int)cudaGetLastError();
}
#endif  // TDS_STEPW_KERNEL_ONLY
