// Model-specialised step kernel: the role-warp kernel of tds_stepr.cu (CTA = a tile of 32 environments x 4 warps,
// warp r = role r of the tree decomposition, lane = environment) instantiated on a COMPILE-TIME model
// (generated/spec_*.h, written by gen_spec.cpp from the flat model).  Joint types, transforms, inertias, collision
// shapes, the decomposition and every index are constant expressions; all loops over links, dofs and contacts are
// unrolled.  What that buys over the table-driven kernel:
//   * straight-line code (no dead branches for absent joint / shape types).  Cold straight-line code is paid at the
//     SM's instruction-fetch rate from L2 (scripts/ifetch_probe.cu on the previous target, not measured on the H100: ~4 cycles / instruction for one stream,
//     ~3.5 for four warps on the SAME stream, 10-12 when four warps stream four different copies), so the four
//     subtrees must be one structural class (Cls below; gen_spec.cpp checks it) and run ONE instruction stream:
//     what differs between them (transforms, axes, inertias, shapes, indices) is read from a per-role table
//     in constant memory; only role 0 additionally runs the trunk code;
//   * per-link state of the subtrees (S, v, c, U, 1/D, u), the mass-matrix blocks M_kk, C -> G and their factors
//     live in registers; shared memory only carries what crosses roles (attachment transforms / accelerations,
//     trunk records, attachment accumulators, partial Schur complements, the trunk factor, contact rows);
//   * massless links, identity transforms and unit axes are folded away;
//   * projected Gauss-Seidel is one warp's work without barriers: role 0 relaxes all rows, in the reference's
//     order, from the contact rows the owners left in shared memory.
// This is the counterpart of the reference's generated cuda_model_<env> (src/utils/cuda_codegen.hpp:156-266),
// with the compiler's constant folding in place of a CppAD operation tape.  Numerics (scalar types RA / RC / RS,
// reference quirks, row order) are those of tds_stept.cu / tds_stepr.cu; citations at each stage.
#include <cuda_runtime.h>
#include <stdlib.h>

#include "tds_wcommon.cuh"
#include "tds_team.h"
#include "generated/spec_laikago.h"
#include "generated/spec_ant.h"

namespace tdss {
using namespace tds;
using namespace tdsw;

#ifndef TDS_DENSE_MAX_CAND
#define TDS_DENSE_MAX_CAND 8   // up to this many contact candidates: every candidate gets a row, unrolled branch-free PGS
#endif
constexpr int TT = TDS_TEAM_T;
constexpr int ST = 32;   // element stride of every shared-memory array: [word][environment]

template <int V> struct IC { static constexpr int value = V; };
// model tables may only be read in constant expressions from device code: force the evaluation
#define CI(...) (IC<(__VA_ARGS__)>::value)
#define CD(...) ([]() { constexpr double cd_v_ = (__VA_ARGS__); return cd_v_; }())
// dot product with a compile-time direction: zero components vanish, +-1 components cost no multiply
#define CDOT3(ax, ay, az, v)                                                                                            \
  ([&]() {                                                                                                              \
    using T_ = decltype((v).x);                                                                                         \
    constexpr double a_ = (ax), b_ = (ay), c_ = (az);                                                                   \
    T_ s_ = T_(-0.0);                                                                                                   \
    if constexpr (a_ == 1.0) s_ += (v).x; else if constexpr (a_ == -1.0) s_ -= (v).x; else if constexpr (a_ != 0.0) s_ += T_(a_) * (v).x; \
    if constexpr (b_ == 1.0) s_ += (v).y; else if constexpr (b_ == -1.0) s_ -= (v).y; else if constexpr (b_ != 0.0) s_ += T_(b_) * (v).y; \
    if constexpr (c_ == 1.0) s_ += (v).z; else if constexpr (c_ == -1.0) s_ -= (v).z; else if constexpr (c_ != 0.0) s_ += T_(c_) * (v).z; \
    return s_;                                                                                                          \
  }())
#define DOT_PN(v) CDOT3(SP::PLANE_N[0], SP::PLANE_N[1], SP::PLANE_N[2], v)
#define DOT_NB(v) CDOT3(-SP::PLANE_N[0], -SP::PLANE_N[1], -SP::PLANE_N[2], v)
#define DOT_F1(v) CDOT3(SP::FR1[0], SP::FR1[1], SP::FR1[2], v)
#define DOT_F2(v) CDOT3(SP::FR2[0], SP::FR2[1], SP::FR2[2], v)
template <int B, int E, class F> TDS_D void sfor(F&& f) {
  if constexpr (B < E) { f(IC<B>{}); sfor<B + 1, E>(f); }
}
template <int B, int E, class F> TDS_D void sfor_rev(F&& f) {   // E-1 down to B
  if constexpr (B < E) { f(IC<E - 1>{}); sfor_rev<B, E - 1>(f); }
}
__host__ __device__ constexpr int cmax(int a, int b) { return a > b ? a : b; }
__host__ __device__ constexpr int ev(int x) { return (x + 1) & ~1; }
__host__ __device__ constexpr int tri(int i, int j) { return i * (i + 1) / 2 + j; }   // i >= j

// is local link j an ancestor of local link k (same role list)?
template <class SP, int R> __host__ __device__ constexpr bool is_anc(int j, int k) {
  for (int a = SP::L_LPAR[R][k]; a >= 0; a = SP::L_LPAR[R][a]) if (a == j) return true;
  return false;
}
template <class SP> __host__ __device__ constexpr int geom_pts(int g) { return SP::G_TYPE[g] == TDSG_SPHERE ? 1 : (SP::G_TYPE[g] == TDSG_CAPSULE ? 2 : 0); }
template <class SP> __host__ __device__ constexpr int pts_before(int g_begin, int g) { int c = 0; for (int i = g_begin; i < g; ++i) c += geom_pts<SP>(i); return c; }
template <class SP, int R> __host__ __device__ constexpr int k_of_q(int q_idx) {   // local link of role R holding coordinate q_idx (-1: none)
  for (int k = 0; k < SP::N_LOC[R]; ++k) if (!(SP::L_FLAGS[R][k] & TDS_LF_FIXED) && SP::L_QIDX[R][k] == q_idx) return k;
  return -1;
}

// Structural class of the four subtrees.  Positions k in [N_TRUNK, N_LOC) of every role's list must agree on
// topology and joint kind; where the roles differ only numerically the class takes the general form
// (joint type -> revolute about a run-time axis, transform -> general) and the numbers come from LegTab.
template <class SP> struct Cls {
  static constexpr int NT = SP::N_TRUNK, NLOC = SP::N_LOC[0], KO = NLOC - NT > 0 ? NLOC - NT : 1;
  static constexpr int STRUCT = TDS_LF_FIXED | TDS_LF_REVOLUTE | TDS_LF_PRISMATIC | TDS_TF_PARENT_ADJ | TDS_TF_CHILD_ADJ | TDS_TF_PARENT_TRUNK;
  __host__ __device__ static constexpr bool zero3(const double* v) { return v[0] == 0.0 && v[1] == 0.0 && v[2] == 0.0; }
  __host__ __device__ static constexpr int flags(int k) {
    int f = SP::L_FLAGS[0][k];
    for (int r = 1; r < SP::T; ++r) if (!(SP::L_FLAGS[r][k] & TDS_LF_XT_IDENT)) f &= ~TDS_LF_XT_IDENT;
    return f;
  }
  __host__ __device__ static constexpr int jtype(int k) {
    int j = SP::L_JTYPE[0][k];
    for (int r = 1; r < SP::T; ++r) if (SP::L_JTYPE[r][k] != j) j = TDSJ_REVOLUTE_AXIS;
    return j;
  }
  __host__ __device__ static constexpr bool massless(int k) {
    for (int r = 0; r < SP::T; ++r) {
      const double* b = SP::L_RBIC[r][k];
      if (!(b[0] == 0.0 && b[4] == 0.0 && b[5] == 0.0 && b[6] == 0.0 && b[7] == 0.0 && b[8] == 0.0 && b[9] == 0.0)) return false;
    }
    return true;
  }
  __host__ __device__ static constexpr bool t_zero(int k) {
    for (int r = 0; r < SP::T; ++r) if (!zero3(&SP::L_XT[r][k][9])) return false;
    return true;
  }
  __host__ __device__ static constexpr bool axis_same(int k) {
    for (int r = 1; r < SP::T; ++r)
      for (int j = 0; j < 3; ++j) if (SP::L_AXIS[r][k][j] != SP::L_AXIS[0][k][j]) return false;
    return true;
  }
  __host__ __device__ static constexpr bool has_sd(int k, int j) {
    for (int r = 0; r < SP::T; ++r) if (SP::L_SD[r][k][j] != 0.0) return true;
    return false;
  }
  __host__ __device__ static constexpr int geom_pts(int g) { return SP::G_TYPE[g] == TDSG_SPHERE ? 1 : (SP::G_TYPE[g] == TDSG_CAPSULE ? 2 : 0); }
  // geoms / candidate points of the subtree, numbered locally in link order (role 0 is the template)
  __host__ __device__ static constexpr int gb_local(int k) { int c = 0; for (int j = NT; j < k; ++j) c += SP::L_GE[0][j] - SP::L_GB[0][j]; return c; }
  __host__ __device__ static constexpr int n_geoms_own() { return gb_local(NLOC); }
  __host__ __device__ static constexpr int gtype_local(int k, int i) { return SP::G_TYPE[SP::L_GB[0][k] + i]; }
  __host__ __device__ static constexpr int pt_local(int k, int i) {   // first point of geom i of link k
    int c = 0;
    for (int j = NT; j <= k; ++j)
      for (int g = SP::L_GB[0][j]; g < (j < k ? SP::L_GE[0][j] : SP::L_GB[0][j] + i); ++g) c += geom_pts(g);
    return c;
  }
  __host__ __device__ static constexpr int n_pts_own() { return pt_local(NLOC - 1, SP::L_GE[0][NLOC - 1] - SP::L_GB[0][NLOC - 1]); }
  __host__ __device__ static constexpr int n_pts_trunk() { return SP::N_PTS[0] - n_pts_own(); }
  __host__ __device__ static constexpr bool uniform() {
    if (NLOC <= NT) return false;
    for (int r = 1; r < SP::T; ++r) {
      if (SP::N_LOC[r] != NLOC || SP::N_OD[r] != SP::N_OD[0] || SP::N_PTS[r] != n_pts_own()) return false;
      for (int k = NT; k < NLOC; ++k) {
        if ((SP::L_FLAGS[r][k] & STRUCT) != (SP::L_FLAGS[0][k] & STRUCT)) return false;
        if (SP::L_LPAR[r][k] != SP::L_LPAR[0][k] || SP::L_LDOF[r][k] != SP::L_LDOF[0][k] || SP::L_ACC[r][k] != SP::L_ACC[0][k] ||
            SP::L_PAR[r][k] != SP::L_PAR[0][k] || SP::L_XW[r][k] != SP::L_XW[0][k]) return false;
        if ((SP::L_ACT[r][k] >= 0) != (SP::L_ACT[0][k] >= 0)) return false;
        if (SP::L_JTYPE[r][k] != SP::L_JTYPE[0][k] && !((SP::L_FLAGS[r][k] & TDS_LF_REVOLUTE) && (SP::L_FLAGS[0][k] & TDS_LF_REVOLUTE))) return false;
        if (SP::L_GE[r][k] - SP::L_GB[r][k] != SP::L_GE[0][k] - SP::L_GB[0][k]) return false;
        for (int i = 0; i < SP::L_GE[0][k] - SP::L_GB[0][k]; ++i)
          if (SP::G_TYPE[SP::L_GB[r][k] + i] != SP::G_TYPE[SP::L_GB[0][k] + i]) return false;
      }
    }
    return true;
  }
};

// What differs between the subtrees: one record per role in constant memory (uniform index -> broadcast loads).
template <class SP> struct LegTab {
  static constexpr int KO = Cls<SP>::KO, NG = Cls<SP>::n_geoms_own() > 0 ? Cls<SP>::n_geoms_own() : 1,
                       NP = Cls<SP>::n_pts_own() > 0 ? Cls<SP>::n_pts_own() : 1;
  double xt[KO][12], axis[KO][3], rbic[KO][10], sd[KO][2];
  double gt[NG][3], ghalf[NG][3], grad[NG];
  int qidx[KO], qdidx[KO], act[KO], link[KO];
  int cand[NP];   // global candidate index of the subtree's p-th point
};
template <class SP> constexpr LegTab<SP> make_leg(int r) {
  using C = Cls<SP>;
  LegTab<SP> t{};
  for (int k = C::NT; k < C::NLOC; ++k) {
    const int o = k - C::NT;
    for (int j = 0; j < 12; ++j) t.xt[o][j] = SP::L_XT[r][k][j];
    for (int j = 0; j < 3; ++j) t.axis[o][j] = SP::L_AXIS[r][k][j];
    for (int j = 0; j < 10; ++j) t.rbic[o][j] = SP::L_RBIC[r][k][j];
    for (int j = 0; j < 2; ++j) t.sd[o][j] = SP::L_SD[r][k][j];
    t.qidx[o] = SP::L_QIDX[r][k]; t.qdidx[o] = SP::L_QDIDX[r][k]; t.act[o] = SP::L_ACT[r][k]; t.link[o] = SP::L_LINK[r][k];
    int p = 0;
    for (int g = SP::L_GB[r][k]; g < SP::L_GE[r][k]; ++g) {
      const int gl = C::gb_local(k) + (g - SP::L_GB[r][k]);
      for (int j = 0; j < 3; ++j) { t.gt[gl][j] = SP::G_T[3 * g + j]; t.ghalf[gl][j] = SP::G_HALF[3 * g + j]; }
      t.grad[gl] = SP::G_RADIUS[g];
      for (int j = 0; j < C::geom_pts(g); ++j) { t.cand[C::pt_local(k, g - SP::L_GB[r][k]) + j] = SP::L_CAND[r][k] + p; ++p; }
    }
  }
  return t;
}
template <class SP> __device__ const LegTab<SP>& leg_tab(int role);

// Trunk links of a CHAIN trunk (every trunk link's parent is the previous one) are swept by run-time loops in the
// leaf->root and root->leaf passes: the loop body is fetched once and then runs out of the instruction caches,
// which beats the unrolled form on a warp that streams alone (role 0).  What the body needs per link:
template <class SP> __host__ __device__ constexpr bool trunk_massless(int k) {
  const double* b = SP::L_RBIC[0][k];
  return b[0] == 0.0 && b[4] == 0.0 && b[5] == 0.0 && b[6] == 0.0 && b[7] == 0.0 && b[8] == 0.0 && b[9] == 0.0;
}
template <class SP> __host__ __device__ constexpr int trunk_rbi_slot(int k) {   // slot among the massive trunk links
  int c = 0;
  for (int j = 0; j < k; ++j) if (!trunk_massless<SP>(j)) ++c;
  return c;
}
template <class SP> struct TrunkTab {
  static constexpr int NTA = SP::N_TRUNK > 0 ? SP::N_TRUNK : 1;
  int fixed[NTA], massless[NTA], acc[NTA], ldof[NTA], qdidx[NTA], xw[NTA], rbi_slot[NTA];
  float sd[NTA][2];
};
template <class SP> __host__ __device__ constexpr bool trunk_is_chain() {
  if (SP::N_TRUNK < 2) return false;
  for (int k = 0; k < SP::N_TRUNK; ++k) {
    if (SP::L_LPAR[0][k] != k - 1) return false;
    if (SP::L_ACC[0][k] >= SP::N_ATT) return false;   // trunk-internal accumulators: not a chain
  }
  return true;
}
// Fixed-base emulation (the reference's locomotion models): a chain of MASSLESS joints carrying one body.  Massless
// links transmit the joint force unchanged in the common frame, so the trunk's forward dynamics is one dense SPD solve
//   (S^T Ia S) qdd = tau - S^T (Ia (a0 + sum_j c_j) + pA),   a_body = a0 + sum_j c_j + S qdd
// with Ia / pA the articulated inertia / bias of the body (own + attached subtrees) -- what the leaf->root sweep of ABA
// computes by six successive rank-1 eliminations of the same matrix.
template <class SP> __host__ __device__ constexpr bool trunk_direct() {
  if (!trunk_is_chain<SP>() || SP::FLOATING) return false;
  for (int k = 0; k < SP::N_TRUNK; ++k) {
    if (SP::L_FLAGS[0][k] & TDS_LF_FIXED) return false;
    if (SP::L_SD[0][k][0] != 0.0 || SP::L_SD[0][k][1] != 0.0) return false;
    if (k < SP::N_TRUNK - 1 && (!trunk_massless<SP>(k) || SP::L_ACC[0][k] >= 0 || SP::L_XW[0][k] >= 0)) return false;
  }
  return true;
}
template <class SP> constexpr TrunkTab<SP> make_trunk() {
  TrunkTab<SP> t{};
  for (int k = 0; k < SP::N_TRUNK; ++k) {
    const double* b = SP::L_RBIC[0][k];
    t.fixed[k] = (SP::L_FLAGS[0][k] & TDS_LF_FIXED) ? 1 : 0;
    t.massless[k] = (b[0] == 0.0 && b[4] == 0.0 && b[5] == 0.0 && b[6] == 0.0 && b[7] == 0.0 && b[8] == 0.0 && b[9] == 0.0) ? 1 : 0;
    t.rbi_slot[k] = trunk_rbi_slot<SP>(k);
    t.acc[k] = SP::L_ACC[0][k]; t.ldof[k] = SP::L_LDOF[0][k]; t.qdidx[k] = SP::L_QDIDX[0][k]; t.xw[k] = SP::L_XW[0][k];
    t.sd[k][0] = (float)SP::L_SD[0][k][0]; t.sd[k][1] = (float)SP::L_SD[0][k][1];
  }
  return t;
}
template <class SP> __device__ const TrunkTab<SP>& trunk_tab();

// contact candidates for the looped Gauss-Seidel sweep (models with many candidates): owner role, has a subtree part
template <class SP> struct CandTab {
  static constexpr int NC = SP::N_CAND > 0 ? SP::N_CAND : 1;
  int owner[NC], own[NC];
};
template <class SP> constexpr CandTab<SP> make_cand() {
  CandTab<SP> t{};
  for (int g = 0; g < SP::N_CAND; ++g) {
    t.owner[g] = SP::CAND_OWNER[g];
    t.own[g] = (SP::CAND_OWNER[g] == 0 && SP::CAND_LPT[g] < Cls<SP>::n_pts_trunk()) ? 0 : 1;
  }
  return t;
}
template <class SP> __device__ const CandTab<SP>& cand_tab();

// shared-memory layout of one tile, 4-byte words per environment
template <class SP, typename RA, typename RC, typename RS> struct Lay {
  static constexpr int RAW = sizeof(RA) / 4, RCW = sizeof(RC) / 4, RSW = sizeof(RS) / 4;
  static constexpr int NTD = SP::N_TD, NTRI = NTD * (NTD + 1) / 2, NOD = SP::N_OD_MAX;
  static constexpr int O = 0;                                        // O[3], plane_off (RC)
  static constexpr int RB = O + 4 * RCW;                             // Rb[9] (RC), floating base
  static constexpr int XWW = ev(12 * RCW + 12 * RAW);                // slot: R[9] p[3] (RC) | v[6] a[6] (RA)
  static constexpr int XW = RB + 10 * RCW;                           // slot 0 = base, then the published trunk links
  static constexpr int TS = XW + (SP::N_XW_TEAM + 1) * XWW;          // trunk S [N_TRUNK][6] (RC)
  static constexpr int TLW = ev(14 * RAW);                           // trunk record: U[6] 1/D u (8 RA) | v/c/a (6 RA)
  static constexpr int TL = TS + SP::N_TRUNK * 6 * RCW;
  static constexpr int TLR = ev(TL + SP::N_TRUNK * TLW);             // rigid inertias (10 RC) of the trunk links that have mass
  static constexpr int TKS = ev(TLR + trunk_rbi_slot<SP>(SP::N_TRUNK) * 10 * RCW);   // per trunk link: q, qd, tau (floats)
  static constexpr int TQD = ev(TKS + 3 * SP::N_TRUNK);              // trunk qd after the FD update (NTD floats)
  static constexpr int ACC_IC = ev(27 * RAW);
  static constexpr int ACCW = ev(ACC_IC + 10 * RCW);                 // attachment accumulator: Ia 21 + pa 6 (RA) | Ic 10 (RC)
  static constexpr int ACC = ev(TQD + NTD);                          // [T][N_ATT]; later the partial Schur complements [T][NTRI] (RS)
  static constexpr int PW = ev(NTRI * RSW);
  static constexpr int CONW = ev((3 * (NOD + NTD) + 9) * RSW);       // contact row: y_own[3][NOD] y_t[3][NTD] b[3] yy[3] 1/A[3]
  // one region, three tenants in time: attachment accumulators (until the trunk sweep), partial Schur complements
  // (until the trunk factorisation), contact rows (from the row phase on); barriers separate the tenants
  static constexpr int ACC_SZ = cmax(cmax(TT * cmax(SP::N_ATT, 1) * ACCW, TT * PW), cmax(SP::N_CAND, 1) * CONW);
  static constexpr int LT = ACC + ACC_SZ;                            // trunk factor, lower triangle with inverted diagonal (RS)
  static constexpr int CON = ACC;                                    // contact rows per candidate (see ACC_SZ)
  static constexpr int ZT = ev(LT + NTRI * RSW);                     // z_t[NTD] (RS)
  static constexpr int WO = ev(ZT + NTD * RSW);                      // w_own[T][NOD] (RS)
  static constexpr int ASTG = ev(WO + TT * NOD * RSW);               // host-layout instance: the tile's actions, linear [env][n_act] floats
  static constexpr int XS = ev(ASTG + SP::N_ACT);                    // impulses x[N_CAND][3] (RS) of the looped PGS sweep
  static constexpr int FLG = ev(XS + (SP::N_CAND > TDS_DENSE_MAX_CAND ? 3 * SP::N_CAND * RSW : 0));   // active masks (2 words per role), done flag
  static constexpr int SHARED = ev(FLG + 2 * TT + 2);
  static constexpr int PRIV = ev(cmax(SP::KMAX - SP::N_TRUNK, 1) * 10 * RCW);   // rigid inertias of the own links (RC)
  static constexpr int TOTAL = SHARED + TT * PRIV;
};

template <typename T> TDS_D T* sp(char* base, int lane, int word) {
  return (sizeof(T) == 4) ? ((T*)base) + (size_t)word * ST + lane : ((T*)base) + (size_t)(word >> 1) * ST + lane;
}
template <typename T> TDS_D T negz() { return T(-0.0); }   // additive identity the optimiser folds exactly
template <typename T> TDS_D Abi<T> abi_nz() {
  Abi<T> a; const T z = negz<T>();
  a.I = {z, z, z, z, z, z}; a.M = a.I;
  a.H.xx = a.H.xy = a.H.xz = a.H.yx = a.H.yy = a.H.yz = a.H.zx = a.H.zy = a.H.zz = z;
  return a;
}
template <typename T> TDS_D Sv<T> sv_nz() { Sv<T> s; const T z = negz<T>(); s.top = v3<T>(z, z, z); s.bot = s.top; return s; }
template <typename T> TDS_D Rbi<T> rbi_nz() { Rbi<T> r; const T z = negz<T>(); r.m = z; r.h = v3<T>(z, z, z); r.I = {z, z, z, z, z, z}; return r; }

// %globaltimer (ns, one clock for the whole device: the gaps between consecutive grids are measured across SMs)
TDS_D long long global_ns() {
#ifdef TDS_STEPS_KERNEL_ONLY   // (the host-compiled copy of the kernel source in tests/cpp has no PTX)
  return 0;
#else
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return (long long)t;
#endif
}

// VAR selects what the instance carries besides the step itself (code bytes are paid at the instruction-fetch rate):
//   0 general: forward-dynamics-only mode, per-link world transforms and contact distances as outputs
//   1 lean: full / no-contact step on the device layout only      2 lean + host layouts (tds_b200_env_step_host)
template <class SP, typename RA, typename RC, typename RS, int VAR>
TDS_D void tile_body(char* const smem, const SimParams& P, const EnvParams& E, const StepIO& io, const int mode, const int use_pd,
                     const int role, const int tile, const int tid) {
  using L = Lay<SP, RA, RC, RS>;
  using C = Cls<SP>;
  static_assert(C::uniform(), "the subtrees of the model are not one structural class (use the table-driven kernel)");
  constexpr bool XOUT = VAR == 0, HOSTIO = VAR == 2;
  constexpr int RAW = L::RAW, RCW = L::RCW;
  constexpr int NT = SP::N_TRUNK, NTD = SP::N_TD, NLOC = SP::N_LOC[0];
  constexpr int NOD = SP::N_OD[0], NODA = cmax(NOD, 1), NTDA = cmax(NTD, 1), NTRI = L::NTRI, NTRIA = cmax(NTRI, 1);
  constexpr int NPO = C::n_pts_own(), NPOA = cmax(NPO, 1), NPTR = C::n_pts_trunk(), NPTRA = cmax(NPTR, 1);
  constexpr int NACCA = cmax(SP::N_ACC, 1), NXLA = cmax(SP::N_XW_LANE, 1), NATT = cmax(SP::N_ATT, 1);
  constexpr bool FLOAT = SP::FLOATING != 0;
  const int lane = tid & 31;
  const int env = tile * 32 + lane;   // (a tile past the end of the batch computes on the last environment and stores nothing)
  const bool live = env < io.n;
  const int e = live ? env : io.n - 1;
  const int ns = io.n_stride;
  const LegTab<SP>& LG = leg_tab<SP>(role);
  char* const priv = smem + (size_t)(L::SHARED + role * L::PRIV) * ST * 4;
  int phase_id = 0;
#define TDSS_PHASE() do { if (io.phase_clk && lane == 0 && tile * 32 < io.n_stride) io.phase_clk[((size_t)tile * TT + role) * 16 + phase_id] = clock64(); ++phase_id; } while (0)
#define TDSS_STAMP(slot) do { if (io.phase_clk && lane == 0 && tile * 32 < io.n_stride) io.phase_clk[((size_t)tile * TT + role) * 16 + (slot)] = clock64(); } while (0)
  TDSS_PHASE();
  auto xw_rc = [&](int slot) { return sp<RC>(smem, lane, L::XW + slot * L::XWW); };                  // R[9], p[3]
  auto xw_ra = [&](int slot) { return sp<RA>(smem, lane, L::XW + slot * L::XWW + 12 * RCW); };       // v[6], a[6]
  auto tl_rbi_slot = [&](int slot) { return sp<RC>(smem, lane, L::TLR + slot * 10 * RCW); };
  auto tl_u = [&](int k) { return sp<RA>(smem, lane, L::TL + k * L::TLW); };
  auto tl_v = [&](int k) { return sp<RA>(smem, lane, L::TL + k * L::TLW + 8 * RAW); };
  auto ts_S = [&](int k) { return sp<RC>(smem, lane, L::TS + k * 6 * RCW); };
  float* const tqd = sp<float>(smem, lane, L::TQD);
  unsigned* const flg = sp<unsigned>(smem, lane, L::FLG);

  // ---- load the coordinates of this role's joints; PD torques (locomotion_contact_simulation.h:168-258) -------------------
  float qv[SP::KMAX], qdv[SP::KMAX], tauv[SP::KMAX];   // joint coordinate / velocity / torque of local link k
  float bq[7], bqd[6];                                 // floating base (role 0)
  sfor<NT, NLOC>([&](auto Kc) {
    constexpr int k = decltype(Kc)::value;
    if constexpr (!(C::flags(k) & TDS_LF_FIXED)) {
      qv[k] = io.q_in[(size_t)LG.qidx[k - NT] * ns + e];
      qdv[k] = io.qd_in[(size_t)LG.qdidx[k - NT] * ns + e];
      tauv[k] = 0.f;
    }
  });
  if (role == 0) {
    sfor<0, NT>([&](auto Kc) {
      constexpr int k = decltype(Kc)::value;
      if constexpr (!(SP::L_FLAGS[0][k] & TDS_LF_FIXED)) {
        qv[k] = io.q_in[(size_t)CI(SP::L_QIDX[0][k]) * ns + e];
        qdv[k] = io.qd_in[(size_t)CI(SP::L_QDIDX[0][k]) * ns + e];
        tauv[k] = 0.f;
      }
    });
    if constexpr (FLOAT) {
#pragma unroll
      for (int k = 0; k < 7; ++k) bq[k] = io.q_in[(size_t)k * ns + e];
#pragma unroll
      for (int k = 0; k < 6; ++k) bqd[k] = io.qd_in[(size_t)k * ns + e];
    }
  }
  // actions: [n_act][n] (device layout); the host-layout instance ([n][n_act], possibly mapped HOST memory read over
  // PCIe) fetches the tile's block with coalesced loads now, parks it in registers during the kinematics pass, stages
  // it in shared memory before the next barrier and computes the PD torques after it
  constexpr int NACT_TILE = 32 * SP::N_ACT, AREG = (NACT_TILE + 32 * TT - 1) / (32 * TT);
  float areg[AREG];
  if constexpr (HOSTIO) {
    const float* const ta = io.act_aos + (size_t)tile * NACT_TILE;
    const int rows = io.n - tile * 32;
    const int valid = (rows < 32 ? rows : 32) * SP::N_ACT;
#pragma unroll
    for (int j = 0; j < AREG; ++j) {
      const int idx = tid + 32 * TT * j;
      areg[j] = idx < valid ? ta[idx] : 0.f;
    }
  }
  float* const astg = (float*)smem + (size_t)L::ASTG * ST;
  const float* const act_p = HOSTIO ? astg + lane * SP::N_ACT : io.tau_in + e;
  const size_t act_s = HOSTIO ? (size_t)1 : (size_t)ns;
  auto pd_torques = [&]() {
    sfor<NT, NLOC>([&](auto Kc) {
      constexpr int k = decltype(Kc)::value;
      if constexpr (!(C::flags(k) & TDS_LF_FIXED) && SP::L_ACT[0][k] >= 0) {
        const int a = LG.act[k - NT];
        float act = act_p[(size_t)a * act_s];
        act = fmaxf(fminf(act, E.action_limit), -E.action_limit);
        const float q_des = E.initial_poses[a] + act;
        const float f = E.kp * (q_des - qv[k]) + E.kd * (0.f - qdv[k]);
        tauv[k] = fminf(fmaxf(f, -E.max_force), E.max_force);
      }
    });
    if (role == 0) {
      sfor<0, NT>([&](auto Kc) {
        constexpr int k = decltype(Kc)::value;
        constexpr int a = SP::L_ACT[0][k];
        if constexpr (!(SP::L_FLAGS[0][k] & TDS_LF_FIXED) && a >= 0) {
          float act = act_p[(size_t)a * act_s];
          act = fmaxf(fminf(act, E.action_limit), -E.action_limit);
          const float q_des = E.initial_poses[a] + act;
          const float f = E.kp * (q_des - qv[k]) + E.kd * (0.f - qdv[k]);
          tauv[k] = fminf(fmaxf(f, -E.max_force), E.max_force);
        }
      });
    }
  };
  if (use_pd) {
    if constexpr (!HOSTIO) pd_torques();
  } else if (io.tau_in) {
    constexpr int off = FLOAT ? 6 : 0;
    sfor<NT, NLOC>([&](auto Kc) {
      constexpr int k = decltype(Kc)::value;
      if constexpr (!(C::flags(k) & TDS_LF_FIXED) && SP::L_QDIDX[0][k] >= off)
        tauv[k] = io.tau_in[(size_t)(LG.qdidx[k - NT] - off) * ns + e];
    });
    if (role == 0) {
      sfor<0, NT>([&](auto Kc) {
        constexpr int k = decltype(Kc)::value;
        if constexpr (!(SP::L_FLAGS[0][k] & TDS_LF_FIXED) && SP::L_QDIDX[0][k] >= off)
          tauv[k] = io.tau_in[(size_t)CI(SP::L_QDIDX[0][k] - off) * ns + e];
      });
    }
  }
  constexpr bool TRUNK_LOOP = trunk_is_chain<SP>();
  // with a looped chain trunk, the rows of the trunk block of M (CRBA) are computed by roles 1.. while role 0 runs the
  // trunk's ABA sweep: they would idle at the barrier otherwise
  constexpr bool CRBA_HELPERS = TRUNK_LOOP && TT > 1;
  constexpr bool DIRECT_TRUNK = trunk_direct<SP>();
  float* const tk_q = sp<float>(smem, lane, L::TKS);
  float* const tk_qd = tk_q + NT * ST;
  float* const tk_tau = tk_qd + NT * ST;
  if constexpr (TRUNK_LOOP) {
    if (role == 0) {
      sfor<0, NT>([&](auto Kc) {
        constexpr int k = decltype(Kc)::value;
        if constexpr (!(SP::L_FLAGS[0][k] & TDS_LF_FIXED)) { tk_q[k * ST] = qv[k]; tk_qd[k * ST] = qdv[k]; tk_tau[k * ST] = tauv[k]; }
      });
    }
  }
  // sines / cosines of every revolute joint of this role up front: independent dependency chains the scheduler can
  // interleave (inside the kinematic chain they would be serialised behind the parent transform)
  RC snv[SP::KMAX], csv[SP::KMAX];
  sfor<NT, NLOC>([&](auto Kc) {
    constexpr int k = decltype(Kc)::value;
    if constexpr ((C::flags(k) & TDS_LF_REVOLUTE) != 0 && !(C::flags(k) & TDS_LF_FIXED))
      sincos_t(CI(C::jtype(k)) == TDSJ_REVOLUTE_AXIS ? RC(qv[k]) * RC(0.5) : RC(qv[k]), &snv[k], &csv[k]);
  });
  if (role == 0) {
    sfor<0, NT>([&](auto Kc) {
      constexpr int k = decltype(Kc)::value;
      if constexpr ((SP::L_FLAGS[0][k] & TDS_LF_REVOLUTE) != 0 && !(SP::L_FLAGS[0][k] & TDS_LF_FIXED))
        sincos_t(CI(SP::L_JTYPE[0][k]) == TDSJ_REVOLUTE_AXIS ? RC(qv[k]) * RC(0.5) : RC(qv[k]), &snv[k], &csv[k]);
    });
  }
  const bool want_contacts = (mode == MODE_FULL) && SP::HAS_PLANE;
  const V3<RC> pn = v3<RC>(RC(CD(SP::PLANE_N[0])), RC(CD(SP::PLANE_N[1])), RC(CD(SP::PLANE_N[2])));
  TDSS_PHASE();  // 1

  // ---- contact candidates (contact_point.hpp:112-116): subtree points (every role) and trunk / base points (role 0) ----------
  unsigned long long my_active = 0ull;   // bit = global candidate index
  V3<RC> cpos[NPOA]; RC cdist[NPOA];     // subtree points, local numbering
  V3<RC> tpos[NPTRA]; RC tdist[NPTRA];   // role 0: points on base / trunk geoms, numbered as in CAND_LPT
  RC plane_off; V3<RC> O;
  auto emit_point = [&](const V3<RC>& pos, const RC rad, const int cand, V3<RC>& out_pos, RC& out_dist) {
    const RC dist = DOT_PN(pos) + plane_off - rad;
    if constexpr (XOUT) if (io.contact_dist && live) io.contact_dist[(size_t)cand * ns + e] = (float)dist;
    out_pos = pos - pn * rad;                                // world_point_on_b, relative to O
    out_dist = dist;
    if (dist < RC(0)) my_active |= 1ull << cand;
  };
  // geoms [gb, ge) of a trunk link / the base (compile-time shapes)
  auto emit_trunk_geoms = [&](auto Gb, auto Ge, auto Cand0, auto Lpt0, const M3<RC>& Rw, const V3<RC>& pw) {
    constexpr int gb = decltype(Gb)::value, ge = decltype(Ge)::value;
    sfor<gb, ge>([&](auto Gc) {
      constexpr int g = decltype(Gc)::value;
      constexpr int ty = SP::G_TYPE[g];
      if constexpr (ty == TDSG_SPHERE || ty == TDSG_CAPSULE) {
        constexpr int cand0 = decltype(Cand0)::value + pts_before<SP>(gb, g), lpt0 = decltype(Lpt0)::value + pts_before<SP>(gb, g);
        const V3<RC> c = pw + mul(Rw, v3<RC>(RC(CD(SP::G_T[3 * g])), RC(CD(SP::G_T[3 * g + 1])), RC(CD(SP::G_T[3 * g + 2]))));
        const RC rad = RC(CD(SP::G_RADIUS[g]));
        if constexpr (ty == TDSG_CAPSULE) {
          const V3<RC> half = mul(Rw, v3<RC>(RC(CD(SP::G_HALF[3 * g])), RC(CD(SP::G_HALF[3 * g + 1])), RC(CD(SP::G_HALF[3 * g + 2]))));
          emit_point(c + half, rad, cand0, tpos[lpt0], tdist[lpt0]);
          emit_point(c - half, rad, cand0 + 1, tpos[lpt0 + 1], tdist[lpt0 + 1]);
        } else emit_point(c, rad, cand0, tpos[lpt0], tdist[lpt0]);
      }
    });
  };
  // geoms of subtree link k (shape types of the class, numbers from the role's table)
  auto emit_own_geoms = [&](auto Kc, const M3<RC>& Rw, const V3<RC>& pw) {
    constexpr int k = decltype(Kc)::value;
    sfor<0, SP::L_GE[0][k] - SP::L_GB[0][k]>([&](auto Ic_) {
      constexpr int i = decltype(Ic_)::value;
      constexpr int ty = C::gtype_local(k, i), gl = C::gb_local(k) + i, p0 = C::pt_local(k, i);
      if constexpr (ty == TDSG_SPHERE || ty == TDSG_CAPSULE) {
        const V3<RC> c = pw + mul(Rw, v3<RC>(RC(LG.gt[gl][0]), RC(LG.gt[gl][1]), RC(LG.gt[gl][2])));
        const RC rad = RC(LG.grad[gl]);
        if constexpr (ty == TDSG_CAPSULE) {
          const V3<RC> half = mul(Rw, v3<RC>(RC(LG.ghalf[gl][0]), RC(LG.ghalf[gl][1]), RC(LG.ghalf[gl][2])));
          emit_point(c + half, rad, LG.cand[p0], cpos[p0], cdist[p0]);
          emit_point(c - half, rad, LG.cand[p0 + 1], cpos[p0 + 1], cdist[p0 + 1]);
        } else emit_point(c, rad, LG.cand[p0], cpos[p0], cdist[p0]);
      }
    });
  };

  // ---- pass 1 on one link (kinematics.hpp:18-148, link.hpp:229-336) in the common frame ---------------------------------------
  // Trunk links (k < N_TRUNK, role 0): every constant is an immediate.  Subtree links: structure from Cls, numbers from LG.
  M3<RC> R_prev; V3<RC> p_prev; Sv<RA> v_prev;                       // carried along chains
  Sv<RC> Sreg[SP::KMAX]; Sv<RA> vreg[SP::KMAX];                      // subtree links: S, then v / c / a
  M3<RC> xwR[NXLA]; V3<RC> xwp[NXLA]; Sv<RA> xwa[NXLA];              // subtree links with non-adjacent children
  auto pass1 = [&](auto Kc) {
    constexpr int k = decltype(Kc)::value;
    constexpr bool TR = k < NT;
    constexpr int ko = TR ? 0 : k - NT;
    constexpr int fl = TR ? SP::L_FLAGS[0][k] : C::flags(k), lpar = SP::L_LPAR[0][k], jt = TR ? SP::L_JTYPE[0][k] : C::jtype(k);
    M3<RC> Rp; V3<RC> pp; Sv<RA> vp;
    if constexpr ((fl & TDS_TF_PARENT_ADJ) != 0) { Rp = R_prev; pp = p_prev; vp = v_prev; }
    else if constexpr (lpar < NT) {      // base (slot 0) or a published trunk link
      constexpr int slot = lpar < 0 ? 0 : SP::L_XW[0][lpar < 0 ? 0 : lpar] + 1;
      static_assert(lpar < 0 || slot >= 1, "parent transform not published");
      Rp = ld9<RC>(xw_rc(slot), ST); pp = ld3<RC>(xw_rc(slot) + 9 * ST, ST); vp = ld6<RA>(xw_ra(slot), ST);
    } else {                             // subtree branch parent
      constexpr int xs = SP::L_XW[0][lpar];
      Rp = xwR[xs]; pp = xwp[xs]; vp = vreg[lpar];
    }
    V3<RC> pi = pp;
    if constexpr (TR) {
      constexpr double tx = SP::L_XT[0][k][9], ty = SP::L_XT[0][k][10], tz = SP::L_XT[0][k][11];
      if constexpr (tx != 0.0 || ty != 0.0 || tz != 0.0) pi = pp + mul(Rp, v3<RC>(RC(tx), RC(ty), RC(tz)));
    } else if constexpr (!C::t_zero(k)) pi = pp + mul(Rp, v3<RC>(RC(LG.xt[ko][9]), RC(LG.xt[ko][10]), RC(LG.xt[ko][11])));
    M3<RC> Ri = Rp;
    if constexpr (!(fl & TDS_LF_XT_IDENT)) {
      M3<RC> r;
      if constexpr (TR) {
        r.xx = RC(CD(SP::L_XT[0][k][0])); r.xy = RC(CD(SP::L_XT[0][k][1])); r.xz = RC(CD(SP::L_XT[0][k][2]));
        r.yx = RC(CD(SP::L_XT[0][k][3])); r.yy = RC(CD(SP::L_XT[0][k][4])); r.yz = RC(CD(SP::L_XT[0][k][5]));
        r.zx = RC(CD(SP::L_XT[0][k][6])); r.zy = RC(CD(SP::L_XT[0][k][7])); r.zz = RC(CD(SP::L_XT[0][k][8]));
      } else {
        r.xx = RC(LG.xt[ko][0]); r.xy = RC(LG.xt[ko][1]); r.xz = RC(LG.xt[ko][2]);
        r.yx = RC(LG.xt[ko][3]); r.yy = RC(LG.xt[ko][4]); r.yz = RC(LG.xt[ko][5]);
        r.zx = RC(LG.xt[ko][6]); r.zy = RC(LG.xt[ko][7]); r.zz = RC(LG.xt[ko][8]);
      }
      Ri = mul(Rp, r);
    }
    Sv<RC> S; S.top = v3<RC>(RC(0), RC(0), RC(0)); S.bot = S.top;
    if constexpr (!(fl & TDS_LF_FIXED)) {
      const RC qi = RC(qv[k]);
      constexpr bool axis_ct = TR || C::axis_same(k);        // axis known at compile time
      constexpr double ax = SP::L_AXIS[0][k][0], ay = SP::L_AXIS[0][k][1], az = SP::L_AXIS[0][k][2];
      V3<RC> axv;
      if constexpr (axis_ct) axv = v3<RC>(RC(ax), RC(ay), RC(az)); else axv = v3<RC>(RC(LG.axis[ko][0]), RC(LG.axis[ko][1]), RC(LG.axis[ko][2]));
      auto rot_axis = [&]() -> V3<RC> {    // Ri * axis, unit axes folded to a column
        if constexpr (axis_ct && ax == 1.0 && ay == 0.0 && az == 0.0) return col_x(Ri);
        else if constexpr (axis_ct && ax == 0.0 && ay == 1.0 && az == 0.0) return col_y(Ri);
        else if constexpr (axis_ct && ax == 0.0 && ay == 0.0 && az == 1.0) return col_z(Ri);
        else return mul(Ri, axv);
      };
      if constexpr ((fl & TDS_LF_PRISMATIC) != 0) {
        const V3<RC> d = rot_axis();
        pi = axpy(d, qi, pi);
        S.bot = d;
      } else {
        const V3<RC> w = rot_axis();
        if constexpr (jt == TDSJ_REVOLUTE_AXIS) {
          const RC dl = sqrt_t(dot(axv, axv));
          RC s = snv[k] / dl;
          const RC c = csv[k];
          Ri = mul(Ri, quat_to_matrix<RC>(axv.x * s, axv.y * s, axv.z * s, c));
        } else {
          const RC s = snv[k], c = csv[k];
          const V3<RC> cx = col_x(Ri), cy = col_y(Ri), cz = col_z(Ri);
          if constexpr (jt == TDSJ_REVOLUTE_X) set_cols(Ri, cx, axpy(cz, s, cy * c), axpy(cy, -s, cz * c));
          else if constexpr (jt == TDSJ_REVOLUTE_Y) set_cols(Ri, axpy(cz, -s, cx * c), cy, axpy(cx, s, cz * c));
          else set_cols(Ri, axpy(cy, s, cx * c), axpy(cx, -s, cy * c), cz);
        }
        S.top = w;
        S.bot = cross(pi, w);
      }
    }
    if constexpr (TR) st6<RC>(ts_S(k), ST, S); else Sreg[k] = S;
    {   // rigid-body inertia about O in world axes (subtree links: private shared memory; massless links: nothing)
      constexpr bool massless = TR ? (SP::L_RBIC[0][k][0] == 0.0 && SP::L_RBIC[0][k][4] == 0.0 && SP::L_RBIC[0][k][5] == 0.0 && SP::L_RBIC[0][k][6] == 0.0 &&
                                      SP::L_RBIC[0][k][7] == 0.0 && SP::L_RBIC[0][k][8] == 0.0 && SP::L_RBIC[0][k][9] == 0.0)
                                   : C::massless(k);
      if constexpr (!massless) {
        double b[10];
        if constexpr (TR) {
          b[0] = CD(SP::L_RBIC[0][k][0]); b[1] = CD(SP::L_RBIC[0][k][1]); b[2] = CD(SP::L_RBIC[0][k][2]); b[3] = CD(SP::L_RBIC[0][k][3]); b[4] = CD(SP::L_RBIC[0][k][4]);
          b[5] = CD(SP::L_RBIC[0][k][5]); b[6] = CD(SP::L_RBIC[0][k][6]); b[7] = CD(SP::L_RBIC[0][k][7]); b[8] = CD(SP::L_RBIC[0][k][8]); b[9] = CD(SP::L_RBIC[0][k][9]);
        } else {
#pragma unroll
          for (int j = 0; j < 10; ++j) b[j] = LG.rbic[ko][j];
        }
        Rbi<RC> r;
        r.m = RC(b[0]);
        const V3<RC> c = pi + mul(Ri, v3<RC>(RC(b[1]), RC(b[2]), RC(b[3])));
        r.h = c * r.m;
        S3<RA> Icf;
        Icf.xx = RA(b[4]); Icf.xy = RA(b[5]); Icf.xz = RA(b[6]); Icf.yy = RA(b[7]); Icf.yz = RA(b[8]); Icf.zz = RA(b[9]);
        const S3<RA> Irot = rot_sym(cvt<RA>(Ri), Icf);
        r.I.xx = RC(Irot.xx); r.I.xy = RC(Irot.xy); r.I.xz = RC(Irot.xz); r.I.yy = RC(Irot.yy); r.I.yz = RC(Irot.yz); r.I.zz = RC(Irot.zz);
        const RC cc = dot(c, c);
        r.I.xx += r.m * (cc - c.x * c.x); r.I.yy += r.m * (cc - c.y * c.y); r.I.zz += r.m * (cc - c.z * c.z);
        r.I.xy -= r.m * c.x * c.y; r.I.xz -= r.m * c.x * c.z; r.I.yz -= r.m * c.y * c.z;
        if constexpr (TR) st_rbi<RC>(tl_rbi_slot(trunk_rbi_slot<SP>(k)), ST, r);
        else st_rbi<RC>(sp<RC>(priv, lane, ko * 10 * RCW), ST, r);
      }
    }
    Sv<RA> v = vp;
    if constexpr (!(fl & TDS_LF_FIXED)) {
      const RA qdi = RA(qdv[k]);
      const Sv<RA> Sf = cvt_sv<RA>(S);
      v.top = axpy(Sf.top, qdi, v.top);
      v.bot = axpy(Sf.bot, qdi, v.bot);
    }
    if constexpr (TR) st6<RA>(tl_v(k), ST, v); else vreg[k] = v;
    constexpr int xs = SP::L_XW[0][k];
    if constexpr (xs >= 0) {
      if constexpr (TR) { st9<RC>(xw_rc(xs + 1), ST, Ri); st3<RC>(xw_rc(xs + 1) + 9 * ST, ST, pi); st6<RA>(xw_ra(xs + 1), ST, v); }
      else { xwR[xs] = Ri; xwp[xs] = pi; }
    }
    if (want_contacts) {
      if constexpr (TR) emit_trunk_geoms(IC<SP::L_GB[0][k]>{}, IC<SP::L_GE[0][k]>{}, IC<SP::L_CAND[0][k]>{}, IC<SP::L_LPT[0][k]>{}, Ri, pi);
      else emit_own_geoms(IC<k>{}, Ri, pi);
    }
    if constexpr (XOUT) if (io.link_xf && live) {
      int link;
      if constexpr (TR) link = CI(SP::L_LINK[0][k]); else link = LG.link[ko];
      float* o = io.link_xf + (size_t)link * 12 * ns + e;
      o[0] = (float)Ri.xx; o[(size_t)1 * ns] = (float)Ri.xy; o[(size_t)2 * ns] = (float)Ri.xz;
      o[(size_t)3 * ns] = (float)Ri.yx; o[(size_t)4 * ns] = (float)Ri.yy; o[(size_t)5 * ns] = (float)Ri.yz;
      o[(size_t)6 * ns] = (float)Ri.zx; o[(size_t)7 * ns] = (float)Ri.zy; o[(size_t)8 * ns] = (float)Ri.zz;
      o[(size_t)9 * ns] = (float)(pi.x + O.x); o[(size_t)10 * ns] = (float)(pi.y + O.y); o[(size_t)11 * ns] = (float)(pi.z + O.z);
    }
    R_prev = Ri; p_prev = pi; v_prev = v;
  };

  // ---- pass 1a: role 0 computes the origin and walks the trunk --------------------------------------------------------------
  RC* const sO = sp<RC>(smem, lane, L::O);
  RC* const sRb = sp<RC>(smem, lane, L::RB);
  if (role == 0) {
    TDSS_STAMP(12);   // role 0: start of pass 1a
    M3<RC> Rb0 = m3_identity<RC>();
    O = v3<RC>(RC(0), RC(0), RC(0));
    if constexpr (FLOAT) {
      Rb0 = quat_to_matrix<RC>(RC(bq[0]), RC(bq[1]), RC(bq[2]), RC(bq[3]));
      O = v3<RC>(RC(bq[4]), RC(bq[5]), RC(bq[6]));
    } else {   // end of the translation-only root chain (links 0..N_PREFIX-1, trunk links in model order)
      M3<RC> Rc = m3_identity<RC>();
      sfor<0, SP::N_PRE>([&](auto Ic_) {
        constexpr int i = decltype(Ic_)::value;
        O = O + mul(Rc, v3<RC>(RC(CD(SP::PRE_XT[12 * i + 9])), RC(CD(SP::PRE_XT[12 * i + 10])), RC(CD(SP::PRE_XT[12 * i + 11]))));
        if constexpr (i < SP::N_PREFIX) {
          static_assert(SP::L_LINK[0][i] == i && i < NT, "root prefix must be trunk links in model order");
          if constexpr (!(SP::PRE_FLAGS[i] & TDS_LF_XT_IDENT)) {
            M3<RC> r;
            r.xx = RC(CD(SP::PRE_XT[12 * i])); r.xy = RC(CD(SP::PRE_XT[12 * i + 1])); r.xz = RC(CD(SP::PRE_XT[12 * i + 2]));
            r.yx = RC(CD(SP::PRE_XT[12 * i + 3])); r.yy = RC(CD(SP::PRE_XT[12 * i + 4])); r.yz = RC(CD(SP::PRE_XT[12 * i + 5]));
            r.zx = RC(CD(SP::PRE_XT[12 * i + 6])); r.zy = RC(CD(SP::PRE_XT[12 * i + 7])); r.zz = RC(CD(SP::PRE_XT[12 * i + 8]));
            Rc = mul(Rc, r);
          }
          if constexpr ((SP::PRE_FLAGS[i] & TDS_LF_PRISMATIC) != 0) {
            const RC qi = RC(qv[i]);
            O = O + mul(Rc, v3<RC>(RC(CD(SP::PRE_AXIS[3 * i])) * qi, RC(CD(SP::PRE_AXIS[3 * i + 1])) * qi, RC(CD(SP::PRE_AXIS[3 * i + 2])) * qi));
          }
        }
      });
    }
    plane_off = DOT_PN(O) - RC(CD(SP::PLANE_C[0]));
    st3<RC>(sO, ST, O); sO[3 * ST] = plane_off;
    if constexpr (FLOAT) st9<RC>(sRb, ST, Rb0);
    R_prev = Rb0;
    p_prev = FLOAT ? v3<RC>(RC(0), RC(0), RC(0)) : v3<RC>(-O.x, -O.y, -O.z);
    if constexpr (FLOAT) {
      const M3<RA> RbA = cvt<RA>(Rb0);
      v_prev.top = mul(RbA, v3<RA>(RA(bqd[0]), RA(bqd[1]), RA(bqd[2])));
      v_prev.bot = mul(RbA, v3<RA>(RA(bqd[3]), RA(bqd[4]), RA(bqd[5])));
    } else { v_prev.top = v3<RA>(RA(0), RA(0), RA(0)); v_prev.bot = v_prev.top; }
    st9<RC>(xw_rc(0), ST, R_prev); st3<RC>(xw_rc(0) + 9 * ST, ST, p_prev); st6<RA>(xw_ra(0), ST, v_prev);
    if (want_contacts) emit_trunk_geoms(IC<SP::GEOM_BEGIN[0]>{}, IC<SP::GEOM_BEGIN[1]>{}, IC<0>{}, IC<0>{}, R_prev, p_prev);
    sfor<0, NT>(pass1);
    TDSS_STAMP(13);   // role 0: end of pass 1a
  }
  __syncthreads();
  // ---- pass 1b: every role walks its subtree --------------------------------------------------------------------------------------
  O = ld3<RC>(sO, ST); plane_off = sO[3 * ST];
  M3<RC> Rb = m3_identity<RC>();
  if constexpr (FLOAT) Rb = ld9<RC>(sRb, ST);
  sfor<NT, NLOC>(pass1);
  // set of active candidates of the environment: OR over the roles through shared memory
  flg[(2 * role) * ST] = (unsigned)my_active;
  flg[(2 * role + 1) * ST] = (unsigned)(my_active >> 32);
  if constexpr (HOSTIO) {
#pragma unroll
    for (int j = 0; j < AREG; ++j) {
      const int idx = tid + 32 * TT * j;
      if (idx < NACT_TILE) astg[idx] = areg[j];
    }
  }
  const bool cta_contact = __syncthreads_or(my_active != 0ull) != 0;   // uniform: any contact in this tile
  if constexpr (HOSTIO) {
    pd_torques();
    if constexpr (TRUNK_LOOP && !DIRECT_TRUNK) {
      if (role == 0) {
        sfor<0, NT>([&](auto Kc) {
          constexpr int k = decltype(Kc)::value;
          if constexpr (!(SP::L_FLAGS[0][k] & TDS_LF_FIXED)) tk_tau[k * ST] = tauv[k];
        });
      }
    }
  }
  const bool solve = (mode == MODE_FULL) && cta_contact;
  unsigned long long team_active = 0ull;
#pragma unroll
  for (int r = 0; r < TT; ++r) team_active |= ((unsigned long long)flg[(2 * r + 1) * ST] << 32) | flg[(2 * r) * ST];
  TDSS_PHASE();  // 2

  // ---- pass 2 on one link: ABA (forward_dynamics.hpp:50-216) + CRBA (mass_matrix.hpp:39-125) ------------------------------------
  // Subtree blocks of the joint-space inertia in registers: M_kk (lower triangle), C = coupling with the trunk dofs;
  // role 0 also holds the trunk block B.
  constexpr int NMKK = NODA * (NODA + 1) / 2, NCM = NODA * NTDA;
  RS Mkk[NMKK];
#ifdef TDS_STEPS_KERNEL_ONLY   // (g++ 13 mis-sizes the capture of this array in the nested generic lambdas of the host-compiled copy)
  RS Cm_store[NCM];
  RS* const Cm = Cm_store;
#else
  RS Cm[NCM];
#endif
  RS Bm[NTRIA];
#pragma unroll
  for (int i = 0; i < NMKK; ++i) Mkk[i] = RS(0);
#pragma unroll
  for (int i = 0; i < NCM; ++i) Cm[i] = RS(0);
#pragma unroll
  for (int i = 0; i < NTRIA; ++i) Bm[i] = RS(0);
  Sv<RA> Ureg[SP::KMAX]; RA invDreg[SP::KMAX], ureg[SP::KMAX];
  Abi<RA> cA = abi_nz<RA>(); Sv<RA> cP = sv_nz<RA>(); Rbi<RC> cC = rbi_nz<RC>();        // carry from the adjacent child
  Abi<RA> accA[NACCA]; Sv<RA> accP[NACCA]; Rbi<RC> accC[NACCA];                          // accumulators (attachment + internal)
#pragma unroll
  for (int s = 0; s < NACCA; ++s) { accA[s] = abi_nz<RA>(); accP[s] = sv_nz<RA>(); accC[s] = rbi_nz<RC>(); }
  auto S_of = [&](auto Jc) -> Sv<RC> {
    constexpr int j = decltype(Jc)::value;
    if constexpr (j < NT) return ld6<RC>(ts_S(j), ST); else return Sreg[j];
  };
  auto acc_ptr_ra = [&](int r, int s) { return sp<RA>(smem, lane, L::ACC + (r * NATT + s) * L::ACCW); };
  auto acc_ptr_rc = [&](int r, int s) { return sp<RC>(smem, lane, L::ACC + (r * NATT + s) * L::ACCW + L::ACC_IC); };
  auto pass2 = [&](auto Kc) {
    constexpr int k = decltype(Kc)::value;
    constexpr bool TR = k < NT;
    constexpr int ko = TR ? 0 : k - NT;
    constexpr int fl = TR ? SP::L_FLAGS[0][k] : C::flags(k);
    constexpr bool massless = TR ? (SP::L_RBIC[0][k][0] == 0.0 && SP::L_RBIC[0][k][4] == 0.0 && SP::L_RBIC[0][k][5] == 0.0 && SP::L_RBIC[0][k][6] == 0.0 &&
                                    SP::L_RBIC[0][k][7] == 0.0 && SP::L_RBIC[0][k][8] == 0.0 && SP::L_RBIC[0][k][9] == 0.0)
                                 : C::massless(k);
    Sv<RA> v;
    if constexpr (TR) v = ld6<RA>(tl_v(k), ST); else v = vreg[k];
    Rbi<RC> Ic = rbi_nz<RC>();
    Abi<RA> Ia = abi_nz<RA>();
    Sv<RA> pA = sv_nz<RA>();
    if constexpr (!massless) {
      if constexpr (TR) Ic = ld_rbi<RC>(tl_rbi_slot(trunk_rbi_slot<SP>(k)), ST); else Ic = ld_rbi<RC>(sp<RC>(priv, lane, ko * 10 * RCW), ST);
      const Rbi<RA> rb = cvt_rbi<RA>(Ic);
      Ia = abi_from_rbi(rb);
      pA = cross_mf(v, rbi_mul(rb, v));                      // kinematics.hpp:132
    }
    if constexpr ((fl & TDS_TF_CHILD_ADJ) != 0) { abi_add(Ia, cA); pA = pA + cP; rbi_add(Ic, cC); }
    constexpr int as = SP::L_ACC[0][k];
    if constexpr (as >= 0) {
      abi_add(Ia, accA[as]); pA = pA + accP[as]; rbi_add(Ic, accC[as]);
      if constexpr (as < SP::N_ATT) {   // attachment slot: role 0's part is in registers, the others' in shared memory
        static_assert(TR || k < 0, "attachment accumulators are consumed by trunk links");
        sfor<1, TT>([&](auto Rc_) {
          constexpr int r = decltype(Rc_)::value;
          Abi<RA> sa; Sv<RA> sv_;
          acc_ld27<RA>(acc_ptr_ra(r, as), ST, sa, sv_);
          abi_add(Ia, sa); pA = pA + sv_;
          rbi_add(Ic, ld_rbi<RC>(acc_ptr_rc(r, as), ST));
        });
      }
    }
    Sv<RA> pa = pA;
    if constexpr (!(fl & TDS_LF_FIXED)) {
      const Sv<RC> Sd = S_of(IC<k>{});
      const Sv<RA> S = cvt_sv<RA>(Sd);
      const RA qdj = RA(qdv[k]);
      Sv<RA> vJ; vJ.top = S.top * qdj; vJ.bot = S.bot * qdj;
      const Sv<RA> c = cross_mm(v, vJ);                      // kinematics.hpp:96-97
      const Sv<RA> U = abi_mul(Ia, S);                       // forward_dynamics.hpp:111
      const RA D = dot(S, U);
      const RA invD = inv_t(D);
      RA tau = RA(tauv[k]);
      if constexpr (TR) {
        if constexpr (SP::L_SD[0][k][0] != 0.0) tau -= RA(CD(SP::L_SD[0][k][0])) * RA(qv[k]);
        if constexpr (SP::L_SD[0][k][1] != 0.0) tau -= RA(CD(SP::L_SD[0][k][1])) * qdj;
      } else {
        if constexpr (C::has_sd(k, 0)) tau -= RA(LG.sd[ko][0]) * RA(qv[k]);
        if constexpr (C::has_sd(k, 1)) tau -= RA(LG.sd[ko][1]) * qdj;
      }
      const RA u = tau - dot(S, pA);                         // :129
      if constexpr (TR) { st6<RA>(tl_v(k), ST, c); st6<RA>(tl_u(k), ST, U); tl_u(k)[6 * ST] = invD; tl_u(k)[7 * ST] = u; }
      else { vreg[k] = c; Ureg[k] = U; invDreg[k] = invD; ureg[k] = u; }
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
      if (solve) {   // CRBA column (mass_matrix.hpp:86-111): M_ij = S_j . (Ic_i S_i)
        const Sv<RC> F = rbi_mul(Ic, Sd);
        const RS mii = RS(dot(Sd, F));
        constexpr int ld = SP::L_LDOF[0][k];
        if constexpr (TR) Bm[tri(ld, ld)] = mii; else Mkk[tri(ld - NTD, ld - NTD)] = mii;
        sfor<0, k>([&](auto Jc) {
          constexpr int j = decltype(Jc)::value;
          constexpr int lj = SP::L_LDOF[0][j];
          if constexpr (lj >= 0 && is_anc<SP, 0>(j, k)) {
            const RS val = RS(dot(S_of(IC<j>{}), F));
            if constexpr (TR) Bm[tri(ld, lj)] = val;
            else if constexpr (lj >= NTD) Mkk[tri(ld - NTD, lj - NTD)] = val;
            else Cm[(ld - NTD) * NTDA + lj] = val;
          }
        });
        if constexpr (FLOAT) {
          const V3<RC> ft = mulT(Rb, F.top), fb = mulT(Rb, F.bot);
          if constexpr (TR) {
            Bm[tri(ld, 0)] = RS(ft.x); Bm[tri(ld, 1)] = RS(ft.y); Bm[tri(ld, 2)] = RS(ft.z);
            Bm[tri(ld, 3)] = RS(fb.x); Bm[tri(ld, 4)] = RS(fb.y); Bm[tri(ld, 5)] = RS(fb.z);
          } else {
            RS* row = Cm + (ld - NTD) * NTDA;
            row[0] = RS(ft.x); row[1] = RS(ft.y); row[2] = RS(ft.z); row[3] = RS(fb.x); row[4] = RS(fb.y); row[5] = RS(fb.z);
          }
        }
      }
    }
    if constexpr ((fl & TDS_TF_PARENT_ADJ) != 0) { cA = Ia; cP = pa; cC = Ic; }
    else {
      constexpr int slot = SP::L_PAR[0][k];
      if constexpr (slot >= 0) { abi_add(accA[slot], Ia); accP[slot] = accP[slot] + pa; rbi_add(accC[slot], Ic); }
    }
  };
  // ---- pass 2a: subtrees; roles 1.. publish their attachment accumulators ------------------------------------------------------------------
  sfor_rev<NT, NLOC>(pass2);
  if (TRUNK_LOOP || role != 0) {
    sfor<0, SP::N_ATT>([&](auto Sc) {
      constexpr int s = decltype(Sc)::value;
      RA* pa_ = acc_ptr_ra(role, s);
      const Abi<RA>& a = accA[s]; const Sv<RA>& f = accP[s];
      pa_[0] = a.I.xx; pa_[ST] = a.I.xy; pa_[2 * ST] = a.I.xz; pa_[3 * ST] = a.I.yy; pa_[4 * ST] = a.I.yz; pa_[5 * ST] = a.I.zz;
      pa_[6 * ST] = a.H.xx; pa_[7 * ST] = a.H.xy; pa_[8 * ST] = a.H.xz; pa_[9 * ST] = a.H.yx; pa_[10 * ST] = a.H.yy; pa_[11 * ST] = a.H.yz;
      pa_[12 * ST] = a.H.zx; pa_[13 * ST] = a.H.zy; pa_[14 * ST] = a.H.zz;
      pa_[15 * ST] = a.M.xx; pa_[16 * ST] = a.M.xy; pa_[17 * ST] = a.M.xz; pa_[18 * ST] = a.M.yy; pa_[19 * ST] = a.M.yz; pa_[20 * ST] = a.M.zz;
      pa_[21 * ST] = f.top.x; pa_[22 * ST] = f.top.y; pa_[23 * ST] = f.top.z; pa_[24 * ST] = f.bot.x; pa_[25 * ST] = f.bot.y; pa_[26 * ST] = f.bot.z;
      st_rbi<RC>(acc_ptr_rc(role, s), ST, accC[s]);
    });
  }
  __syncthreads();
  TDSS_STAMP(10);   // end of pass 2a (all roles, after the barrier)

  // ---- pass 2b + base + pass 3a: role 0 finishes the trunk --------------------------------------------------------------------------------
  const RA dtA = RA(P.dt);
  Sv<RA> a_prev;
  auto pass3 = [&](auto Kc) {
    constexpr int k = decltype(Kc)::value;
    constexpr bool TR = k < NT;
    constexpr int ko = TR ? 0 : k - NT;
    constexpr int fl = TR ? SP::L_FLAGS[0][k] : C::flags(k), lpar = SP::L_LPAR[0][k];
    Sv<RA> a;
    if constexpr ((fl & TDS_TF_PARENT_ADJ) != 0) a = a_prev;
    else if constexpr (lpar < NT) {
      constexpr int slot = lpar < 0 ? 0 : SP::L_XW[0][lpar < 0 ? 0 : lpar] + 1;
      a = ld6<RA>(xw_ra(slot) + 6 * ST, ST);
    } else a = xwa[CI(SP::L_XW[0][lpar < NT ? NT : lpar])];
    if constexpr (!(fl & TDS_LF_FIXED)) {
      Sv<RA> c, U; RA invD, u;
      if constexpr (TR) { c = ld6<RA>(tl_v(k), ST); U = ld6<RA>(tl_u(k), ST); invD = tl_u(k)[6 * ST]; u = tl_u(k)[7 * ST]; }
      else { c = vreg[k]; U = Ureg[k]; invD = invDreg[k]; u = ureg[k]; }
      a = a + c;
      const RA qdd = invD * (u - dot(U, a));
      const Sv<RA> S = cvt_sv<RA>(S_of(IC<k>{}));
      a.top = axpy(S.top, qdd, a.top);
      a.bot = axpy(S.bot, qdd, a.bot);
      if (XOUT && mode == MODE_FD) {
        if (live && io.qdd_out) {
          int qdi;
          if constexpr (TR) qdi = CI(SP::L_QDIDX[0][k]); else qdi = LG.qdidx[ko];
          io.qdd_out[(size_t)qdi * ns + e] = (float)qdd;
        }
      } else qdv[k] = (float)(RA(qdv[k]) + qdd * dtA);
    }
    constexpr int xs = SP::L_XW[0][k];
    if constexpr (xs >= 0) {
      if constexpr (TR) st6<RA>(xw_ra(xs + 1) + 6 * ST, ST, a); else xwa[xs] = a;
    }
    a_prev = a;
  };
  if constexpr (CRBA_HELPERS) {
    if (role != 0 && solve) {
      const TrunkTab<SP>& TK = trunk_tab<SP>();
      RS* const Bs = sp<RS>(smem, lane, L::LT);
      Rbi<RC> Ic = rbi_nz<RC>();   // composite inertia of the chain from link k to the leaves
#pragma unroll 1
      for (int k = NT - 1; k >= 0; --k) {
        if (!TK.massless[k]) rbi_add(Ic, ld_rbi<RC>(tl_rbi_slot(TK.rbi_slot[k]), ST));
        const int as = TK.acc[k];
        if (as >= 0) {
#pragma unroll
          for (int r = 0; r < TT; ++r) rbi_add(Ic, ld_rbi<RC>(acc_ptr_rc(r, as), ST));
        }
        if (!TK.fixed[k] && (k % (TT - 1)) == role - 1) {   // rows are dealt round-robin to roles 1..
          const Sv<RC> Sd = ld6<RC>(ts_S(k), ST);
          const Sv<RC> F = rbi_mul(Ic, Sd);
          const int ld = TK.ldof[k];
          RS* const brow = Bs + (size_t)(ld * (ld + 1) / 2) * ST;
          brow[ld * ST] = RS(dot(Sd, F));
#pragma unroll
          for (int j = 0; j < NT - 1; ++j) {
            const int lj = TK.ldof[j];
            if (j < k && lj >= 0) brow[lj * ST] = RS(dot(ld6<RC>(ts_S(j), ST), F));
          }
          if constexpr (FLOAT) {
            const V3<RC> ft = mulT(Rb, F.top), fb = mulT(Rb, F.bot);
            brow[0] = RS(ft.x); brow[ST] = RS(ft.y); brow[2 * ST] = RS(ft.z);
            brow[3 * ST] = RS(fb.x); brow[4 * ST] = RS(fb.y); brow[5 * ST] = RS(fb.z);
          }
        }
      }
    }
  }
  if (role == 0) {
    if constexpr (DIRECT_TRUNK) {
      // (massless chain trunk: solved in one piece below, after the base acceleration)
    } else if constexpr (TRUNK_LOOP) {
      // chain trunk, leaf -> root, run-time loop (same arithmetic as pass2 above; state in shared memory)
      const TrunkTab<SP>& TK = trunk_tab<SP>();
      RS* const Bs = sp<RS>(smem, lane, L::LT);   // trunk block of M, lower triangle (factorised in place later)
      cA = abi_nz<RA>(); cP = sv_nz<RA>(); cC = rbi_nz<RC>();
#pragma unroll 1
      for (int k = NT - 1; k >= 0; --k) {
        const Sv<RA> v = ld6<RA>(tl_v(k), ST);
        Rbi<RC> Ic = cC; Abi<RA> Ia = cA; Sv<RA> pA = cP;
        if (!TK.massless[k]) {
          const Rbi<RC> own = ld_rbi<RC>(tl_rbi_slot(TK.rbi_slot[k]), ST);
          const Rbi<RA> rb = cvt_rbi<RA>(own);
          abi_add(Ia, abi_from_rbi(rb));
          pA = pA + cross_mf(v, rbi_mul(rb, v));
          rbi_add(Ic, own);
        }
        const int as = TK.acc[k];
        if (as >= 0) {
#pragma unroll
          for (int r = 0; r < TT; ++r) {
            Abi<RA> sa; Sv<RA> sv_;
            acc_ld27<RA>(acc_ptr_ra(r, as), ST, sa, sv_);
            abi_add(Ia, sa); pA = pA + sv_;
            rbi_add(Ic, ld_rbi<RC>(acc_ptr_rc(r, as), ST));
          }
        }
        Sv<RA> pa = pA;
        if (!TK.fixed[k]) {
          const Sv<RC> Sd = ld6<RC>(ts_S(k), ST);
          const Sv<RA> S = cvt_sv<RA>(Sd);
          const RA qdj = RA(tk_qd[k * ST]);
          Sv<RA> vJ; vJ.top = S.top * qdj; vJ.bot = S.bot * qdj;
          const Sv<RA> c = cross_mm(v, vJ);
          const Sv<RA> U = abi_mul(Ia, S);
          const RA D = dot(S, U);
          const RA invD = inv_t(D);
          RA tau = RA(tk_tau[k * ST]);
          tau -= RA(TK.sd[k][0]) * RA(tk_q[k * ST]);
          tau -= RA(TK.sd[k][1]) * qdj;
          const RA u = tau - dot(S, pA);
          st6<RA>(tl_v(k), ST, c); st6<RA>(tl_u(k), ST, U); tl_u(k)[6 * ST] = invD; tl_u(k)[7 * ST] = u;
          const V3<RA> ut = U.top * invD, ub = U.bot * invD;
          Ia.I.xx -= U.top.x * ut.x; Ia.I.xy -= U.top.x * ut.y; Ia.I.xz -= U.top.x * ut.z;
          Ia.I.yy -= U.top.y * ut.y; Ia.I.yz -= U.top.y * ut.z; Ia.I.zz -= U.top.z * ut.z;
          Ia.H.xx -= U.top.x * ub.x; Ia.H.xy -= U.top.x * ub.y; Ia.H.xz -= U.top.x * ub.z;
          Ia.H.yx -= U.top.y * ub.x; Ia.H.yy -= U.top.y * ub.y; Ia.H.yz -= U.top.y * ub.z;
          Ia.H.zx -= U.top.z * ub.x; Ia.H.zy -= U.top.z * ub.y; Ia.H.zz -= U.top.z * ub.z;
          Ia.M.xx -= U.bot.x * ub.x; Ia.M.xy -= U.bot.x * ub.y; Ia.M.xz -= U.bot.x * ub.z;
          Ia.M.yy -= U.bot.y * ub.y; Ia.M.yz -= U.bot.y * ub.z; Ia.M.zz -= U.bot.z * ub.z;
          const Sv<RA> Iac = abi_mul(Ia, c);
          const RA uD = u * invD;
          pa.top = pA.top + Iac.top + U.top * uD;
          pa.bot = pA.bot + Iac.bot + U.bot * uD;
          if (solve && !CRBA_HELPERS) {   // CRBA column: the ancestors of a chain link are all the links before it
            const Sv<RC> F = rbi_mul(Ic, Sd);
            const int ld = TK.ldof[k];
            RS* const brow = Bs + (size_t)(ld * (ld + 1) / 2) * ST;
            brow[ld * ST] = RS(dot(Sd, F));
#pragma unroll
            for (int j = 0; j < NT - 1; ++j) {   // unrolled: independent dot products, static addresses
              const int lj = TK.ldof[j];
              if (j < k && lj >= 0) brow[lj * ST] = RS(dot(ld6<RC>(ts_S(j), ST), F));
            }
            if constexpr (FLOAT) {
              const V3<RC> ft = mulT(Rb, F.top), fb = mulT(Rb, F.bot);
              brow[0] = RS(ft.x); brow[ST] = RS(ft.y); brow[2 * ST] = RS(ft.z);
              brow[3 * ST] = RS(fb.x); brow[4 * ST] = RS(fb.y); brow[5 * ST] = RS(fb.z);
            }
          }
        }
        cA = Ia; cP = pa; cC = Ic;
      }
    } else sfor_rev<0, NT>(pass2);
    TDSS_STAMP(11);   // role 0: end of the trunk's leaf->root pass
    // base acceleration (forward_dynamics.hpp:218-243)
    Sv<RC> base_acc_b; base_acc_b.top = v3<RC>(RC(0), RC(0), RC(0)); base_acc_b.bot = base_acc_b.top;
    if constexpr (FLOAT) {
      Abi<RA> Ach = abi_nz<RA>(); Sv<RA> pch = sv_nz<RA>(); Rbi<RC> Icch = rbi_nz<RC>();
      if constexpr (NT > 0) {
        if constexpr (SP::L_LPAR[0][0] < 0 && (SP::L_FLAGS[0][0] & TDS_TF_PARENT_ADJ) != 0) { abi_add(Ach, cA); pch = pch + cP; rbi_add(Icch, cC); }
      }
      if constexpr (SP::BASE_SLOT >= 0) {
        constexpr int as = SP::BASE_SLOT;
        abi_add(Ach, accA[as]); pch = pch + accP[as]; rbi_add(Icch, accC[as]);
        if constexpr (as < SP::N_ATT) {
          sfor<1, TT>([&](auto Rc_) {
            constexpr int r = decltype(Rc_)::value;
            Abi<RA> sa; Sv<RA> sv_;
            acc_ld27<RA>(acc_ptr_ra(r, as), ST, sa, sv_);
            abi_add(Ach, sa); pch = pch + sv_;
            rbi_add(Icch, ld_rbi<RC>(acc_ptr_rc(r, as), ST));
          });
        }
      }
      const M3<RA> Rt = cvt<RA>(transpose(Rb));
      Abi<RA> Ab;
      {
        Rbi<RA> rbb; rbb.m = RA(CD(SP::BASE_RBI[0])); rbb.h = v3<RA>(RA(CD(SP::BASE_RBI[1])), RA(CD(SP::BASE_RBI[2])), RA(CD(SP::BASE_RBI[3])));
        rbb.I = {RA(CD(SP::BASE_RBI[4])), RA(CD(SP::BASE_RBI[5])), RA(CD(SP::BASE_RBI[6])), RA(CD(SP::BASE_RBI[7])), RA(CD(SP::BASE_RBI[8])), RA(CD(SP::BASE_RBI[9]))};
        Ab = abi_from_rbi(rbb);
        Abi<RA> Arot;
        Arot.I = rot_sym(Rt, Ach.I); Arot.M = rot_sym(Rt, Ach.M); Arot.H = rot_gen(Rt, Ach.H);
        abi_add(Ab, Arot);
      }
      Sv<RA> pb;
      {   // gyroscopic bias, kinematics.hpp:54-61
        const M3<RA> RbA = cvt<RA>(Rb);
        M3<RA> Ic0;
        Ic0.xx = RA((float)CD(SP::BASE_INERTIA_COM[0])); Ic0.xy = RA((float)CD(SP::BASE_INERTIA_COM[1])); Ic0.xz = RA((float)CD(SP::BASE_INERTIA_COM[2]));
        Ic0.yx = RA((float)CD(SP::BASE_INERTIA_COM[3])); Ic0.yy = RA((float)CD(SP::BASE_INERTIA_COM[4])); Ic0.yz = RA((float)CD(SP::BASE_INERTIA_COM[5]));
        Ic0.zx = RA((float)CD(SP::BASE_INERTIA_COM[6])); Ic0.zy = RA((float)CD(SP::BASE_INERTIA_COM[7])); Ic0.zz = RA((float)CD(SP::BASE_INERTIA_COM[8]));
        const M3<RA> Iw = rot_gen(RbA, Ic0);
        const V3<RA> wb = v3<RA>(RA(bqd[0]), RA(bqd[1]), RA(bqd[2]));
        pb.top = cross(wb, mul(Iw, wb)) + mul(Rt, pch.top);
        pb.bot = mul(Rt, pch.bot);
      }
      if (solve) {   // base block of M (mass_matrix.hpp:114-120) in the base frame
        Rbi<RC> Ib; Ib.m = RC(CD(SP::BASE_RBI[0])); Ib.h = v3<RC>(RC(CD(SP::BASE_RBI[1])), RC(CD(SP::BASE_RBI[2])), RC(CD(SP::BASE_RBI[3])));
        Ib.I = {RC(CD(SP::BASE_RBI[4])), RC(CD(SP::BASE_RBI[5])), RC(CD(SP::BASE_RBI[6])), RC(CD(SP::BASE_RBI[7])), RC(CD(SP::BASE_RBI[8])), RC(CD(SP::BASE_RBI[9]))};
        const M3<RC> RtC = transpose(Rb);
        Rbi<RC> rot; rot.m = Icch.m; rot.h = mul(RtC, Icch.h); rot.I = rot_sym(RtC, Icch.I);
        rbi_add(Ib, rot);
        const RS z = RS(0);
        Bm[tri(0, 0)] = RS(Ib.I.xx); Bm[tri(1, 0)] = RS(Ib.I.xy); Bm[tri(1, 1)] = RS(Ib.I.yy);
        Bm[tri(2, 0)] = RS(Ib.I.xz); Bm[tri(2, 1)] = RS(Ib.I.yz); Bm[tri(2, 2)] = RS(Ib.I.zz);
        Bm[tri(3, 0)] = z;            Bm[tri(3, 1)] = RS(Ib.h.z);  Bm[tri(3, 2)] = RS(-Ib.h.y);
        Bm[tri(4, 0)] = RS(-Ib.h.z);  Bm[tri(4, 1)] = z;           Bm[tri(4, 2)] = RS(Ib.h.x);
        Bm[tri(5, 0)] = RS(Ib.h.y);   Bm[tri(5, 1)] = RS(-Ib.h.x); Bm[tri(5, 2)] = z;
        Bm[tri(3, 3)] = RS(Ib.m); Bm[tri(4, 3)] = z; Bm[tri(4, 4)] = RS(Ib.m); Bm[tri(5, 3)] = z; Bm[tri(5, 4)] = z; Bm[tri(5, 5)] = RS(Ib.m);
      }
      {   // -base_abi.inv_mul(bias) with the reference's block inverse (C = -H), inertia.hpp:302-328
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
        M3<RC> Cn = neg(H3);
        M3<RC> Dm = inv3(sub(M3m, mul(mul(Cn, Ainv), H3)));
        M3<RC> AinvBD = mul(mul(Ainv, H3), Dm);
        M3<RC> Ii = add(Ainv, mul(mul(AinvBD, Cn), Ainv));
        M3<RC> Hi = neg(AinvBD);
        V3<RC> ft = cvt<RC>(pb.top), fb = cvt<RC>(pb.bot);
        V3<RC> at = mul(Ii, ft) + mul(Hi, fb);
        V3<RC> ab = mul(Dm, fb) + mulT(Hi, ft);
        base_acc_b.top = v3<RC>(-at.x, -at.y, -at.z);
        base_acc_b.bot = v3<RC>(-ab.x, -ab.y, -ab.z);
      }
      a_prev.top = cvt<RA>(mul(Rb, base_acc_b.top));
      a_prev.bot = cvt<RA>(mul(Rb, base_acc_b.bot));
    } else {
      a_prev.top = v3<RA>(RA(0), RA(0), RA(0));
      a_prev.bot = v3<RA>(RA(-P.gravity[0]), RA(-P.gravity[1]), RA(-P.gravity[2]));
    }
    st6<RA>(xw_ra(0) + 6 * ST, ST, a_prev);
    if constexpr (DIRECT_TRUNK) {
      constexpr int kb = NT - 1;   // the body
      const Sv<RA> v_b = ld6<RA>(tl_v(kb), ST);
      Abi<RA> Ia = abi_nz<RA>(); Sv<RA> pA = sv_nz<RA>();
      if constexpr (!trunk_massless<SP>(kb)) {
        const Rbi<RA> rb = cvt_rbi<RA>(ld_rbi<RC>(tl_rbi_slot(trunk_rbi_slot<SP>(kb)), ST));
        Ia = abi_from_rbi(rb);
        pA = cross_mf(v_b, rbi_mul(rb, v_b));                  // kinematics.hpp:132
      }
      constexpr int as = SP::L_ACC[0][kb];
      if constexpr (as >= 0) {
        sfor<0, TT>([&](auto Rc_) {
          constexpr int r = decltype(Rc_)::value;
          Abi<RA> sa; Sv<RA> sv_;
          acc_ld27<RA>(acc_ptr_ra(r, as), ST, sa, sv_);
          abi_add(Ia, sa); pA = pA + sv_;
        });
      }
      Sv<RA> Sk[NT], Uk[NT];
      Sv<RA> acc = a_prev;                                       // a0 + sum_j c_j
      sfor<0, NT>([&](auto Kc) {
        constexpr int k = decltype(Kc)::value;
        Sk[k] = cvt_sv<RA>(ld6<RC>(ts_S(k), ST));
        const RA qdk = RA(qdv[k]);
        Sv<RA> vJ; vJ.top = Sk[k].top * qdk; vJ.bot = Sk[k].bot * qdk;
        acc = acc + cross_mm(ld6<RA>(tl_v(k), ST), vJ);          // kinematics.hpp:96-97
        Uk[k] = abi_mul(Ia, Sk[k]);                              // forward_dynamics.hpp:111
      });
      const Sv<RA> w = abi_mul(Ia, acc) + pA;
      // (the sweep it replaces eliminates the same matrix in RA arithmetic, one pivot per link)
      RA Dm[NT * (NT + 1) / 2], x[NT];
      sfor<0, NT>([&](auto Ic_) {
        constexpr int i = decltype(Ic_)::value;
        x[i] = RA(tauv[i]) - dot(Sk[i], w);
        sfor<0, i + 1>([&](auto Jc) { constexpr int j = decltype(Jc)::value; Dm[tri(i, j)] = dot(Sk[i], Uk[j]); });
      });
      // D = L L^T (diagonal stored inverted), L y = rhs, L^T qdd = y
      sfor<0, NT>([&](auto Ic_) {
        constexpr int i = decltype(Ic_)::value;
        sfor<0, i + 1>([&](auto Jc) {
          constexpr int j = decltype(Jc)::value;
          RA sacc = Dm[tri(i, j)];
          sfor<0, j>([&](auto Kc) { constexpr int k = decltype(Kc)::value; sacc -= Dm[tri(i, k)] * Dm[tri(j, k)]; });
          if constexpr (j < i) Dm[tri(i, j)] = sacc * Dm[tri(j, j)];
          else Dm[tri(i, i)] = rsqrt_t(sacc);
        });
        RA sy = x[i];
        sfor<0, i>([&](auto Kc) { constexpr int k = decltype(Kc)::value; sy -= Dm[tri(i, k)] * x[k]; });
        x[i] = sy * Dm[tri(i, i)];
      });
      sfor_rev<0, NT>([&](auto Ic_) {
        constexpr int i = decltype(Ic_)::value;
        RA sy = x[i];
        sfor<i + 1, NT>([&](auto Kc) { constexpr int k = decltype(Kc)::value; sy -= Dm[tri(k, i)] * x[k]; });
        x[i] = sy * Dm[tri(i, i)];
      });
      Sv<RA> a = acc;
      sfor<0, NT>([&](auto Kc) {
        constexpr int k = decltype(Kc)::value;
        const RA qdd = x[k];
        a.top = axpy(Sk[k].top, qdd, a.top);
        a.bot = axpy(Sk[k].bot, qdd, a.bot);
        if (XOUT && mode == MODE_FD) { if (live && io.qdd_out) io.qdd_out[(size_t)CI(SP::L_QDIDX[0][k]) * ns + e] = (float)qdd; }
        else qdv[k] = (float)(RA(qdv[k]) + qdd * dtA);
      });
      constexpr int xsb = SP::L_XW[0][kb];
      if constexpr (xsb >= 0) st6<RA>(xw_ra(xsb + 1) + 6 * ST, ST, a);
      a_prev = a;
    } else if constexpr (TRUNK_LOOP) {
      const TrunkTab<SP>& TK = trunk_tab<SP>();
      Sv<RA> a = a_prev;
#pragma unroll 1
      for (int k = 0; k < NT; ++k) {
        if (!TK.fixed[k]) {
          const Sv<RA> c = ld6<RA>(tl_v(k), ST), U = ld6<RA>(tl_u(k), ST);
          const RA invD = tl_u(k)[6 * ST], u = tl_u(k)[7 * ST];
          a = a + c;
          const RA qdd = invD * (u - dot(U, a));
          const Sv<RA> S = cvt_sv<RA>(ld6<RC>(ts_S(k), ST));
          a.top = axpy(S.top, qdd, a.top);
          a.bot = axpy(S.bot, qdd, a.bot);
          if (XOUT && mode == MODE_FD) { if (live && io.qdd_out) io.qdd_out[(size_t)TK.qdidx[k] * ns + e] = (float)qdd; }
          else tk_qd[k * ST] = (float)(RA(tk_qd[k * ST]) + qdd * dtA);
        }
        const int xs = TK.xw[k];
        if (xs >= 0) st6<RA>(xw_ra(xs + 1) + 6 * ST, ST, a);
      }
      a_prev = a;
      sfor<0, NT>([&](auto Kc) {
        constexpr int k = decltype(Kc)::value;
        if constexpr (!(SP::L_FLAGS[0][k] & TDS_LF_FIXED)) qdv[k] = tk_qd[k * ST];
      });
    } else sfor<0, NT>(pass3);
    if constexpr (FLOAT) {   // forward_dynamics.hpp:317-322 (gravity added un-rotated), integrator.hpp:153-163
      const RC qb[6] = {base_acc_b.top.x, base_acc_b.top.y, base_acc_b.top.z, base_acc_b.bot.x + RC(P.gravity[0]),
                        base_acc_b.bot.y + RC(P.gravity[1]), base_acc_b.bot.z + RC(P.gravity[2])};
#pragma unroll
      for (int k = 0; k < 6; ++k) {
        if (XOUT && mode == MODE_FD) { if (live && io.qdd_out) io.qdd_out[(size_t)k * ns + e] = (float)qb[k]; }
        else bqd[k] = (float)(RC(bqd[k]) + qb[k] * RC(P.dt));
      }
#pragma unroll
      for (int k = 0; k < 6; ++k) tqd[k * ST] = bqd[k];
    }
    // publish the updated trunk velocities (contact Jacobian products of every role)
    sfor<0, NT>([&](auto Kc) {
      constexpr int k = decltype(Kc)::value;
      if constexpr (SP::L_LDOF[0][k] >= 0) tqd[CI(SP::L_LDOF[0][k]) * ST] = qdv[k];
    });
  }
  __syncthreads();
  TDSS_PHASE();  // 3
  // ---- pass 3b: subtrees -----------------------------------------------------------------------------------------------------------------------
  sfor<NT, NLOC>(pass3);
  TDSS_PHASE();  // 4
  if (XOUT && mode == MODE_FD) return;

  // ---- contact solve: leaf-first elimination in registers ---------------------------------------------------------------------------------------
  //   M_kk = L_k L_k^T, G = L_k^-1 C, S = B - sum_k G^T G = L_t L_t^T, Y = L^-1 Jc^T, PGS on w = Y p, dqd = L^-T w
  //   (mb_constraint_solver.hpp:299-345, 417-436, 476-497).  Diagonal entries hold the INVERSE of the factor's diagonal.
  if (solve) {
    sfor<0, NOD>([&](auto Ic_) {
      constexpr int i = decltype(Ic_)::value;
      sfor<0, i + 1>([&](auto Jc) {
        constexpr int j = decltype(Jc)::value;
        RS s = Mkk[tri(i, j)];
        sfor<0, j>([&](auto Kc) { constexpr int k = decltype(Kc)::value; s -= Mkk[tri(i, k)] * Mkk[tri(j, k)]; });
        if constexpr (j < i) Mkk[tri(i, j)] = s * Mkk[tri(j, j)];
        else Mkk[tri(i, i)] = rsqrt_t(s);
      });
      sfor<0, NTD>([&](auto Tc) {
        constexpr int t = decltype(Tc)::value;
        RS s = Cm[i * NTDA + t];
        sfor<0, i>([&](auto Kc) { constexpr int k = decltype(Kc)::value; s -= Mkk[tri(i, k)] * Cm[k * NTDA + t]; });
        Cm[i * NTDA + t] = s * Mkk[tri(i, i)];
      });
    });
    // partial Schur complement of this role -> shared memory (the accumulator region is free now)
    RS* const Pk = sp<RS>(smem, lane, L::ACC + role * L::PW);
    sfor<0, NTD>([&](auto T1) {
      constexpr int t1 = decltype(T1)::value;
      sfor<0, t1 + 1>([&](auto T2) {
        constexpr int t2 = decltype(T2)::value;
        RS s = RS(0);
        sfor<0, NOD>([&](auto Ic_) { constexpr int i = decltype(Ic_)::value; s += Cm[i * NTDA + t1] * Cm[i * NTDA + t2]; });
        Pk[tri(t1, t2) * ST] = s;
      });
    });
    __syncthreads();
    RS* const Lt = sp<RS>(smem, lane, L::LT);
    if (role == 0) {   // S = B - sum over the roles of G^T G, then S = L_t L_t^T
      if constexpr (TRUNK_LOOP) {   // rows of the trunk links were written to shared memory by the run-time loop
        sfor<(FLOAT ? 6 : 0), NTD>([&](auto Ic_) {
          constexpr int i = decltype(Ic_)::value;
          sfor<0, i + 1>([&](auto Jc) { constexpr int j = decltype(Jc)::value; Bm[tri(i, j)] = Lt[tri(i, j) * ST]; });
        });
      }
      sfor<0, NTRI>([&](auto Ic_) {
        constexpr int i = decltype(Ic_)::value;
        const RS* p = sp<RS>(smem, lane, L::ACC);
        Bm[i] -= (p[i * ST] + p[(L::PW / L::RSW + i) * ST]) + (p[(2 * (L::PW / L::RSW) + i) * ST] + p[(3 * (L::PW / L::RSW) + i) * ST]);
      });
      sfor<0, NTD>([&](auto Ic_) {
        constexpr int i = decltype(Ic_)::value;
        sfor<0, i + 1>([&](auto Jc) {
          constexpr int j = decltype(Jc)::value;
          RS s = Bm[tri(i, j)];
          sfor<0, j>([&](auto Kc) { constexpr int k = decltype(Kc)::value; s -= Bm[tri(i, k)] * Bm[tri(j, k)]; });
          if constexpr (j < i) Bm[tri(i, j)] = s * Bm[tri(j, j)];
          else Bm[tri(i, i)] = rsqrt_t(s);
          Lt[tri(i, j) * ST] = Bm[tri(i, j)];
        });
      });
    }
    __syncthreads();
  }
  TDSS_PHASE();  // 5
  constexpr int YT = 3 * L::NOD, BB = 3 * (L::NOD + L::NTD);   // row layout: y_own | y_t | b[3] yy[3] 1/A[3]
  // Few candidates: every candidate gets a row (zeros when it does not penetrate: x stays 0) and the sweep below is
  // branch-free straight-line code; many candidates: only penetrating points are visited.
  constexpr bool DENSE = SP::N_CAND <= TDS_DENSE_MAX_CAND;
  if (solve) {
    // contact directions: world_normal_on_b = -plane normal, friction directions from plane_space (compile-time constants)
    const RS* const Lt = sp<RS>(smem, lane, L::LT);
    // contact rows of one penetrating point on local link kl (-1: base): normal, friction 1, friction 2
    auto zero_row = [&](const int cand) {
      RS* const row = sp<RS>(smem, lane, L::CON) + (size_t)cand * (L::CONW / L::RSW) * ST;
#pragma unroll
      for (int i = 0; i < BB + 9; ++i) row[i * ST] = RS(0);
    };
    auto point_rows = [&](auto Kl, const int cand, const V3<RC>& xc, const RC dist) {
      constexpr int kl = decltype(Kl)::value;
      RS ro[3][NODA], rt[3][NTDA];
#pragma unroll
      for (int d = 0; d < 3; ++d) {
#pragma unroll
        for (int i = 0; i < NODA; ++i) ro[d][i] = RS(0);
#pragma unroll
        for (int i = 0; i < NTDA; ++i) rt[d][i] = RS(0);
      }
      V3<RC> vel = v3<RC>(RC(0), RC(0), RC(0));
      if constexpr (FLOAT) {   // jacobian.hpp:39-58 with r = x_c
        const V3<RC> cols[6] = {v3<RC>(RC(0), -xc.z, xc.y), v3<RC>(xc.z, RC(0), -xc.x), v3<RC>(-xc.y, xc.x, RC(0)),
                                v3<RC>(RC(1), RC(0), RC(0)), v3<RC>(RC(0), RC(1), RC(0)), v3<RC>(RC(0), RC(0), RC(1))};
#pragma unroll
        for (int k = 0; k < 6; ++k) {
          rt[0][k] = RS(DOT_NB(cols[k])); rt[1][k] = RS(DOT_F1(cols[k])); rt[2][k] = RS(DOT_F2(cols[k]));
          vel = vel + cols[k] * RC(tqd[k * ST]);
        }
      }
      sfor<0, (kl < 0 ? 0 : kl + 1)>([&](auto Jc) {   // jacobian.hpp:63-80: the link and its ancestors
        constexpr int j = decltype(Jc)::value;
        constexpr int lj = SP::L_LDOF[0][j];
        if constexpr (lj >= 0 && (j == kl || is_anc<SP, 0>(j, kl))) {
          const Sv<RC> S = S_of(IC<j>{});
          const V3<RC> col = S.bot + cross(S.top, xc);
          const RS c0 = RS(DOT_NB(col)), c1 = RS(DOT_F1(col)), c2 = RS(DOT_F2(col));
          if constexpr (lj >= NTD) { ro[0][lj - NTD] = c0; ro[1][lj - NTD] = c1; ro[2][lj - NTD] = c2; vel = vel + col * RC(qdv[j]); }
          else { rt[0][lj] = c0; rt[1][lj] = c1; rt[2][lj] = c2; vel = vel + col * RC(tqd[lj * ST]); }
        }
      });
      RS* const row = sp<RS>(smem, lane, L::CON) + (size_t)cand * (L::CONW / L::RSW) * ST;
      row[(BB + 0) * ST] = RS((RC(1) + RC(P.restitution)) * DOT_NB(vel) - RC(P.erp) * dist * RC(P.inv_dt));
      row[(BB + 1) * ST] = RS(DOT_F1(vel));
      row[(BB + 2) * ST] = RS(DOT_F2(vel));
#pragma unroll
      for (int d = 0; d < 3; ++d) {
        // y_own = L_k^-1 r_own ;  y_t = L_t^-1 (r_t - G^T y_own)   (a trunk point has no own part)
        RS yy = RS(0);
        if constexpr (kl >= NT) {
          sfor<0, NOD>([&](auto Ic_) {
            constexpr int i = decltype(Ic_)::value;
            RS s = ro[d][i];
            sfor<0, i>([&](auto Kc) { constexpr int k = decltype(Kc)::value; s -= Mkk[tri(i, k)] * ro[d][k]; });
            ro[d][i] = s * Mkk[tri(i, i)];
          });
        }
        sfor<0, NOD>([&](auto Ic_) { constexpr int i = decltype(Ic_)::value; yy += ro[d][i] * ro[d][i]; row[(d * L::NOD + i) * ST] = ro[d][i]; });
        sfor<0, NTD>([&](auto Tc) {
          constexpr int t = decltype(Tc)::value;
          RS s = rt[d][t];
          if constexpr (kl >= NT) sfor<0, NOD>([&](auto Ic_) { constexpr int i = decltype(Ic_)::value; s -= Cm[i * NTDA + t] * ro[d][i]; });
          sfor<0, t>([&](auto Kc) { constexpr int k = decltype(Kc)::value; s -= Lt[tri(t, k) * ST] * rt[d][k]; });
          rt[d][t] = s * Lt[tri(t, t) * ST];
          yy += rt[d][t] * rt[d][t];
          row[(YT + d * L::NTD + t) * ST] = rt[d][t];
        });
        // A_ii = y.y + cfm is constant during the sweep: keep y.y and 1 / A_ii per row
        row[(BB + 3 + d) * ST] = yy;
        row[(BB + 6 + d) * ST] = inv_t(yy + RS(P.cfm));
      }
    };
    // subtree points (every role)
    sfor<NT, NLOC>([&](auto Kc) {
      constexpr int k = decltype(Kc)::value;
      sfor<0, SP::L_GE[0][k] - SP::L_GB[0][k]>([&](auto Ic_) {
        constexpr int i = decltype(Ic_)::value;
        sfor<0, C::geom_pts(SP::L_GB[0][k] + i)>([&](auto Jc) {
          constexpr int p = C::pt_local(k, i) + decltype(Jc)::value;
          const int cand = LG.cand[p];
          if ((my_active >> cand) & 1ull) point_rows(IC<k>{}, cand, cpos[p], cdist[p]);
          else if constexpr (DENSE) zero_row(cand);
        });
      });
    });
    // base / trunk points (role 0)
    if (role == 0) {
      auto trunk_rows = [&](auto Kl, auto Gb, auto Ge, auto Cand0, auto Lpt0) {
        constexpr int gb = decltype(Gb)::value, ge = decltype(Ge)::value;
        sfor<gb, ge>([&](auto Gc) {
          constexpr int g = decltype(Gc)::value;
          sfor<0, geom_pts<SP>(g)>([&](auto Jc) {
            constexpr int cand = decltype(Cand0)::value + pts_before<SP>(gb, g) + decltype(Jc)::value;
            constexpr int lpt = decltype(Lpt0)::value + pts_before<SP>(gb, g) + decltype(Jc)::value;
            if ((my_active >> cand) & 1ull) point_rows(Kl, cand, tpos[lpt], tdist[lpt]);
            else if constexpr (DENSE) zero_row(cand);
          });
        });
      };
      trunk_rows(IC<-1>{}, IC<SP::GEOM_BEGIN[0]>{}, IC<SP::GEOM_BEGIN[1]>{}, IC<0>{}, IC<0>{});
      sfor<0, NT>([&](auto Kc) {
        constexpr int k = decltype(Kc)::value;
        trunk_rows(IC<k>{}, IC<SP::L_GB[0][k]>{}, IC<SP::L_GE[0][k]>{}, IC<SP::L_CAND[0][k]>{}, IC<SP::L_LPT[0][k]>{});
      });
    }
    __syncthreads();
  }
  TDSS_PHASE();  // 6
  if (solve) {
    RS* const zt = sp<RS>(smem, lane, L::ZT);
    RS* const wo_s = sp<RS>(smem, lane, L::WO);
    if (role == 0) {
      // projected Gauss-Seidel in the reference's row order (solve_pgs, mb_constraint_solver.hpp:101-142,417-436):
      // blocks normal | friction 1 | friction 2, contacts in enumeration order.  w = Y p stays in registers.
      const RS* const Lt = sp<RS>(smem, lane, L::LT);
      constexpr int NODM = L::NOD, NODMA = cmax(NODM, 1), NCA = cmax(SP::N_CAND, 1);
      RS wt[NTDA], wo[TT][NODMA], x[NCA][3];
#pragma unroll
      for (int i = 0; i < NTDA; ++i) wt[i] = RS(0);
#pragma unroll
      for (int r = 0; r < TT; ++r)
#pragma unroll
        for (int i = 0; i < NODMA; ++i) wo[r][i] = RS(0);
#pragma unroll
      for (int g = 0; g < NCA; ++g) { x[g][0] = RS(0); x[g][1] = RS(0); x[g][2] = RS(0); }
      const RS mu = RS(P.friction);
      if constexpr (!DENSE) {
        // many candidates: run-time loop over the rows (body fetched once), impulses and subtree parts of w in shared
        // memory, only penetrating candidates are visited
        const CandTab<SP>& CT = cand_tab<SP>();
        RS* const xs = sp<RS>(smem, lane, L::XS);
        for (int i = 0; i < 3 * SP::N_CAND; ++i) xs[i * ST] = RS(0);
        for (int i = 0; i < TT * NODM; ++i) wo_s[i * ST] = RS(0);
        for (int it = 0; it < P.pgs_iterations; ++it) {
          sfor<0, 3>([&](auto Dc) {
            constexpr int d = decltype(Dc)::value;
#pragma unroll 1
            for (int g = 0; g < SP::N_CAND; ++g) {
              if (!((team_active >> g) & 1ull)) continue;
              const RS* const row = sp<RS>(smem, lane, L::CON) + (size_t)g * (L::CONW / L::RSW) * ST;
              RS* const wog = wo_s + (size_t)CT.owner[g] * NODM * ST;
              const bool own = CT.own[g] != 0;
              RS yo[NODMA], yt[NTDA];
              RS yw = RS(0);
              sfor<0, NODM>([&](auto Ic_) { constexpr int i = decltype(Ic_)::value; yo[i] = own ? row[(d * L::NOD + i) * ST] : RS(0); yw += yo[i] * wog[i * ST]; });
              sfor<0, NTD>([&](auto Tc) { constexpr int t = decltype(Tc)::value; yt[t] = row[(YT + d * L::NTD + t) * ST]; yw += yt[t] * wt[t]; });
              const RS x_old = xs[(3 * g + d) * ST];
              RS xn = (row[(BB + d) * ST] - yw + row[(BB + 3 + d) * ST] * x_old) * row[(BB + 6 + d) * ST];
              if constexpr (d == 0) {
                xn = xn < RS(0) ? RS(0) : xn;
                xn = xn > RS(100000) ? RS(100000) : xn;
              } else {
                RS sn = xs[(3 * g) * ST];
                sn = sn < RS(0) ? RS(0) : sn;
                const RS lim = mu * sn;
                xn = xn < -lim ? -lim : xn;
                xn = xn > lim ? lim : xn;
              }
              xs[(3 * g + d) * ST] = xn;
              const RS dx = xn - x_old;
              sfor<0, NODM>([&](auto Ic_) { constexpr int i = decltype(Ic_)::value; wog[i * ST] += dx * yo[i]; });
              sfor<0, NTD>([&](auto Tc) { constexpr int t = decltype(Tc)::value; wt[t] += dx * yt[t]; });
            }
          });
        }
      } else
      for (int it = 0; it < P.pgs_iterations; ++it) {
        sfor<0, 3>([&](auto Dc) {
          constexpr int d = decltype(Dc)::value;
          sfor<0, SP::N_CAND>([&](auto Gc) {
            constexpr int g = decltype(Gc)::value;
            constexpr int owner = SP::CAND_OWNER[g];
            // a point on a trunk / base geom has no subtree part
            constexpr bool own_part = !(owner == 0 && SP::CAND_LPT[g] < NPTR);
            constexpr int nod = own_part ? NOD : 0;
            if (DENSE || ((team_active >> g) & 1ull)) {
              const RS* const row = sp<RS>(smem, lane, L::CON + g * L::CONW);
              RS yo[cmax(nod, 1)], yt[NTDA];
              RS yw = RS(0);
              sfor<0, nod>([&](auto Ic_) { constexpr int i = decltype(Ic_)::value; yo[i] = row[(d * L::NOD + i) * ST]; yw += yo[i] * wo[owner][i]; });
              sfor<0, NTD>([&](auto Tc) { constexpr int t = decltype(Tc)::value; yt[t] = row[(YT + d * L::NTD + t) * ST]; yw += yt[t] * wt[t]; });
              const RS x_old = x[g][d];
              RS xn = (row[(BB + d) * ST] - yw + row[(BB + 3 + d) * ST] * x_old) * row[(BB + 6 + d) * ST];
              if constexpr (d == 0) {
                xn = xn < RS(0) ? RS(0) : xn;
                xn = xn > RS(100000) ? RS(100000) : xn;
              } else {
                RS s = x[g][0];
                s = s < RS(0) ? RS(0) : s;
                const RS lim = mu * s;
                xn = xn < -lim ? -lim : xn;
                xn = xn > lim ? lim : xn;
              }
              x[g][d] = xn;
              const RS dx = xn - x_old;
              sfor<0, nod>([&](auto Ic_) { constexpr int i = decltype(Ic_)::value; wo[owner][i] += dx * yo[i]; });
              sfor<0, NTD>([&](auto Tc) { constexpr int t = decltype(Tc)::value; wt[t] += dx * yt[t]; });
            }
          });
        });
      }
      // z_t = L_t^-T w_t ; publish z_t and every role's w_own
      sfor_rev<0, NTD>([&](auto Ic_) {
        constexpr int i = decltype(Ic_)::value;
        RS s = wt[i];
        sfor<i + 1, NTD>([&](auto Kc) { constexpr int k = decltype(Kc)::value; s -= Lt[tri(k, i) * ST] * wt[k]; });
        wt[i] = s * Lt[tri(i, i) * ST];
        zt[i * ST] = wt[i];
      });
      if constexpr (DENSE) {
#pragma unroll
        for (int r = 0; r < TT; ++r)
#pragma unroll
          for (int i = 0; i < NODM; ++i) wo_s[(r * NODM + i) * ST] = wo[r][i];
      }
    }
    __syncthreads();
    TDSS_PHASE();  // 7
    {   // z_k = L_k^-T (w_k - G z_t) ; qd -= z
      RS w[NODA], z[NTDA];
      sfor<0, NTD>([&](auto Tc) { constexpr int t = decltype(Tc)::value; z[t] = zt[t * ST]; });
      sfor<0, NOD>([&](auto Ic_) {
        constexpr int i = decltype(Ic_)::value;
        RS s = wo_s[(role * L::NOD + i) * ST];
        sfor<0, NTD>([&](auto Tc) { constexpr int t = decltype(Tc)::value; s -= Cm[i * NTDA + t] * z[t]; });
        w[i] = s;
      });
      sfor_rev<0, NOD>([&](auto Ic_) {
        constexpr int i = decltype(Ic_)::value;
        RS s = w[i];
        sfor<i + 1, NOD>([&](auto Kc) { constexpr int k = decltype(Kc)::value; s -= Mkk[tri(k, i)] * w[k]; });
        w[i] = s * Mkk[tri(i, i)];
      });
      sfor<NT, NLOC>([&](auto Kc) {
        constexpr int k = decltype(Kc)::value;
        constexpr int lj = SP::L_LDOF[0][k];
        if constexpr (lj >= 0) qdv[k] = (float)(RS(qdv[k]) - w[lj - NTD]);
      });
      if (role == 0) {
        if constexpr (FLOAT) {
#pragma unroll
          for (int k = 0; k < 6; ++k) bqd[k] = (float)(RS(bqd[k]) - z[k]);
        }
        sfor<0, NT>([&](auto Kc) {
          constexpr int k = decltype(Kc)::value;
          constexpr int lj = SP::L_LDOF[0][k];
          if constexpr (lj >= 0) qdv[k] = (float)(RS(qdv[k]) - z[lj]);
        });
      }
    }
  } else { TDSS_PHASE(); }
  TDSS_PHASE();  // 8

  // ---- integrate_euler with qdd = 0 (integrator.hpp:10-133), reward / done, write back ---------------------------------------------------
  sfor<NT, NLOC>([&](auto Kc) {
    constexpr int k = decltype(Kc)::value;
    if constexpr (!(C::flags(k) & TDS_LF_FIXED)) qv[k] = (float)(RC(qv[k]) + RC(qdv[k]) * RC(P.dt));
  });
  if (role == 0) {
    RC up_z = RC(1);
    if constexpr (FLOAT) {
      const RC h = RC(0.5) * RC(P.dt);
      RC qx = RC(bq[0]), qy = RC(bq[1]), qz = RC(bq[2]), qw = RC(bq[3]);
      const RC w0 = RC(bqd[0]), w1 = RC(bqd[1]), w2 = RC(bqd[2]);
      const RC dw = (-qx * w0 - qy * w1 - qz * w2) * h;
      const RC dx = (qw * w0 + qz * w1 - qy * w2) * h;
      const RC dy = (qw * w1 + qx * w2 - qz * w0) * h;
      const RC dz = (qw * w2 + qy * w0 - qx * w1) * h;
      qx += dx; qy += dy; qz += dz; qw += dw;
      const RC len = sqrt_t(qx * qx + qy * qy + qz * qz + qw * qw);
      qx /= len; qy /= len; qz /= len; qw /= len;
      bq[0] = (float)qx; bq[1] = (float)qy; bq[2] = (float)qz; bq[3] = (float)qw;
#pragma unroll
      for (int k = 0; k < 3; ++k) bq[4 + k] = (float)(RC(bq[4 + k]) + RC(bqd[3 + k]) * RC(P.dt));
      up_z = RC(1) - RC(2) * (qx * qx + qy * qy) / (qx * qx + qy * qy + qz * qz + qw * qw);
    }
    sfor<0, NT>([&](auto Kc) {
      constexpr int k = decltype(Kc)::value;
      if constexpr (!(SP::L_FLAGS[0][k] & TDS_LF_FIXED)) qv[k] = (float)(RC(qv[k]) + RC(qdv[k]) * RC(P.dt));
    });
    bool done = false;
    float rew = 0.f;
    if (E.reward_kind == 1) {   // laikago_environment2.h:130-171 (fixed-base emulation; q0..5 are trunk coordinates)
      constexpr int k0 = k_of_q<SP, 0>(0), k2 = k_of_q<SP, 0>(2), k3 = k_of_q<SP, 0>(3), k4 = k_of_q<SP, 0>(4);
      if constexpr (!FLOAT && k0 >= 0 && k0 < NT && k2 >= 0 && k2 < NT && k3 >= 0 && k3 < NT && k4 >= 0 && k4 < NT) {
        const float x = qv[k0], z = qv[k2];
        const float upz = cosf(qv[k3]) * cosf(qv[k4]);
        done = (upz < 0.6f) || (z < 0.2f);
        rew = done ? 0.f : x;
        if (io.reward && live) io.reward[e] = rew;
      }
    } else if (E.reward_kind == 3) {   // ant_environment2.h:75-105: done = z < 0.26, reward = (x' - x)/dt, which integrate_euler makes the x velocity
      constexpr int k0 = k_of_q<SP, 0>(0), k2 = k_of_q<SP, 0>(2);
      if constexpr (!FLOAT && k0 >= 0 && k0 < NT && k2 >= 0 && k2 < NT) {
        done = qv[k2] < 0.26f;
        rew = done ? 0.f : qdv[k0];
        if (io.reward && live) io.reward[e] = rew;
      }
    } else if (E.reward_kind == 2) {
      if constexpr (FLOAT) {
        const float x = bq[4], z = bq[6];
        done = ((float)up_z < 0.6f) || (z < 0.2f);
        rew = done ? 0.f : x;
        if (io.reward && live) io.reward[e] = rew;
      }
    }
    if (io.done && E.reward_kind && live) io.done[e] = done ? 1.f : 0.f;
    if constexpr (HOSTIO) if (io.obs_tail && live) { io.obs_tail[e] = rew; io.obs_tail[io.n + e] = done ? 1.f : 0.f; }
    flg[(2 * TT) * ST] = done ? 1u : 0u;
  }
  __syncthreads();
  const bool reset = (flg[(2 * TT) * ST] != 0u) && E.auto_reset;
  // host-layout instance: the tile's observation block [env][n_q + n_qd] is assembled in shared memory (the contact-row
  // region is free now) and written with coalesced stores - the destination may be mapped host memory
  float* const ostg = (float*)smem + (size_t)L::ACC * ST;
  static_assert(!HOSTIO || (SP::N_Q + SP::N_QD) <= L::ACC_SZ, "observation staging does not fit the reused region");
  if (live) {
    sfor<NT, NLOC>([&](auto Kc) {
      constexpr int k = decltype(Kc)::value;
      if constexpr (!(C::flags(k) & TDS_LF_FIXED)) {
        const int qi = LG.qidx[k - NT], qdi = LG.qdidx[k - NT];
        const float qo = reset ? E.reset_q[qi] : qv[k], qdo = reset ? 0.f : qdv[k];
        io.q_out[(size_t)qi * ns + e] = qo;
        io.qd_out[(size_t)qdi * ns + e] = qdo;
        if constexpr (HOSTIO) { float* o = ostg + lane * (SP::N_Q + SP::N_QD); o[qi] = qo; o[SP::N_Q + qdi] = qdo; }
      }
    });
    if (role == 0) {
      sfor<0, NT>([&](auto Kc) {
        constexpr int k = decltype(Kc)::value;
        if constexpr (!(SP::L_FLAGS[0][k] & TDS_LF_FIXED)) {
          const float qo = reset ? E.reset_q[CI(SP::L_QIDX[0][k])] : qv[k], qdo = reset ? 0.f : qdv[k];
          io.q_out[(size_t)CI(SP::L_QIDX[0][k]) * ns + e] = qo;
          io.qd_out[(size_t)CI(SP::L_QDIDX[0][k]) * ns + e] = qdo;
          if constexpr (HOSTIO) { float* o = ostg + lane * (SP::N_Q + SP::N_QD); o[CI(SP::L_QIDX[0][k])] = qo; o[SP::N_Q + CI(SP::L_QDIDX[0][k])] = qdo; }
        }
      });
      if constexpr (FLOAT) {
#pragma unroll
        for (int k = 0; k < 7; ++k) {
          const float qo = reset ? E.reset_q[k] : bq[k];
          io.q_out[(size_t)k * ns + e] = qo;
          if constexpr (HOSTIO) ostg[lane * (SP::N_Q + SP::N_QD) + k] = qo;
        }
#pragma unroll
        for (int k = 0; k < 6; ++k) {
          const float qdo = reset ? 0.f : bqd[k];
          io.qd_out[(size_t)k * ns + e] = qdo;
          if constexpr (HOSTIO) ostg[lane * (SP::N_Q + SP::N_QD) + SP::N_Q + k] = qdo;
        }
      }
    }
  }
  if constexpr (HOSTIO) {
    if (io.obs_aos) {
      __syncthreads();
      constexpr int NOBS = SP::N_Q + SP::N_QD;
      const int rows = io.n - tile * 32;
      const int valid = (rows < 32 ? rows : 32) * NOBS;
      float* const dst = io.obs_aos + (size_t)tile * 32 * NOBS;
      if (valid == 32 * NOBS && (NOBS % 4) == 0) {
        for (int i = tid; i < 8 * NOBS; i += 32 * TT) ((float4*)dst)[i] = ((const float4*)ostg)[i];
      } else {
        for (int i = tid; i < valid; i += 32 * TT) dst[i] = ostg[i];
      }
    }
  }
  TDSS_PHASE();  // 9
  // %globaltimer after the role's last store (slot 15; slot 14 is stamped by the kernel around griddepcontrol.wait)
  if (io.phase_clk && lane == 0 && tile * 32 < io.n_stride) io.phase_clk[((size_t)tile * TT + role) * 16 + 15] = global_ns();
#undef TDSS_PHASE
#undef TDSS_STAMP
}

// Warms L2 with the rows of global memory the tile reads first: q, qd and the device-layout actions / torques, 128 B
// (32 environments) per row, one row per thread.  Runs BEFORE griddepcontrol.wait, i.e. possibly while the previous
// kernel of the stream (the previous step, a policy kernel) still writes these rows: a prefetch only moves lines into
// L2, the GPU's point of coherence, and returns nothing to the SM; the loads that feed the arithmetic stay after the
// wait.  The host-layout actions may be mapped host memory and are not prefetched.
template <class SP, int VAR> TDS_D void prefetch_tile_rows(const StepIO& io, const int use_pd, const int tile, const int tid) {
  constexpr int NA = VAR == 2 ? 0 : SP::N_ACT, NTAU = VAR == 2 ? 0 : SP::N_QD - (SP::FLOATING ? 6 : 0);
  const int n_in = io.tau_in ? (use_pd ? NA : NTAU) : 0;
  const size_t col = (size_t)tile * 32;
  const float* row = nullptr;
  if (tid < SP::N_Q) row = io.q_in + (size_t)tid * io.n_stride;
  else if (tid < SP::N_Q + SP::N_QD) row = io.qd_in + (size_t)(tid - SP::N_Q) * io.n_stride;
  else if (tid < SP::N_Q + SP::N_QD + n_in) row = io.tau_in + (size_t)(tid - SP::N_Q - SP::N_QD) * io.n_stride;
#ifndef TDS_STEPS_KERNEL_ONLY
  if (row) asm volatile("prefetch.global.L2 [%0];" :: "l"(row + col));
#endif
}

// TPC tiles per CTA.  1 (shipped): one tile per CTA, two CTAs may share an SM.
// 2 (experiment, -DTDS_B200_WITH_TPC2 + TDS_B200_TPC=2): two tiles in one CTA of 8 warps with shared barriers, so that both
// run ONE instruction stream (scripts/icache_probe.cu: two streams over 100+ KB of code pay 3.7-4.6 cycles per instruction
// each, one stream 2.6).  Measured SLOWER (65536 envs: 0.63 vs 0.68 G env-steps/s): in lockstep both tiles sit in their
// single-warp serial sections at the same time, while independent CTAs drift apart and fill each other's idle slots.
template <class SP, typename RA, typename RC, typename RS, int VAR, int TPC>
__global__ void __launch_bounds__(32 * TDS_TEAM_T * TPC, TPC == 1 ? 2 : 1)
tds_step_spec_kernel(const __grid_constant__ SimParams P, const __grid_constant__ EnvParams E, const StepIO io, const int mode_flags,
                     const int use_pd) {
  extern __shared__ __align__(16) char smem_raw[];
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);   // warp index, known uniform to the compiler
  const int role = warp % TDS_TEAM_T, sub = warp / TDS_TEAM_T;
  if ((mode_flags & 256) && role != 0) return;   // profiling aid (TDS_B200_DEBUG_SOLO): role 0 alone, results are garbage
  const int tile = (int)blockIdx.x * TPC + sub, tid = (int)threadIdx.x - sub * 32 * TDS_TEAM_T;
  char* const smem = smem_raw + (size_t)sub * ((size_t)Lay<SP, RA, RC, RS>::TOTAL * 32 * 4);
  // profiling: %globaltimer stamps in the free slots of the (tile, role) record: slot 14 = kernel entry (role 0) or the
  // return from griddepcontrol.wait (roles 1..), slot 15 = after the role's last store (end of tile_body)
  long long* const gstamp = (io.phase_clk && (tid & 31) == 0 && tile * 32 < io.n_stride) ? io.phase_clk + ((size_t)tile * TDS_TEAM_T + role) * 16 : nullptr;
  if (gstamp && role == 0) gstamp[14] = global_ns();
  // Programmatic dependent launch (launched with cudaLaunchAttributeProgrammaticStreamSerialization, SpecHost::launch):
  // with mode bit 512 (a single-wave grid) the next step's grid may be scheduled from now on; its CTAs take the SMs this
  // grid leaves idle or vacates and run up to their own wait.  Everything above the wait reads nothing that earlier work in the
  // stream writes; griddepcontrol.wait returns once the previous grid has completed and its memory is visible.
#ifndef TDS_STEPS_KERNEL_ONLY
  if (mode_flags & 512) asm volatile("griddepcontrol.launch_dependents;");
#endif
  prefetch_tile_rows<SP, VAR>(io, use_pd, tile, tid);
#ifndef TDS_STEPS_KERNEL_ONLY
  asm volatile("griddepcontrol.wait;" ::: "memory");
#endif
  if (gstamp && role != 0) gstamp[14] = global_ns();
  tile_body<SP, RA, RC, RS, VAR>(smem, P, E, io, mode_flags & 255, use_pd, role, tile, tid);
#ifndef TDS_STEPS_KERNEL_ONLY
  if (!(mode_flags & 512)) asm volatile("griddepcontrol.launch_dependents;");
#endif
}

#ifndef TDS_STEPS_KERNEL_ONLY   // launchers / registry: not part of the host-compiled kernel source (tests/cpp/steps_host.cpp)
template <class SP> struct SpecHost {
  static bool matches(const DevModel* D, const EnvParams* E) {
    if (D->n_links != SP::N_LINKS || D->n_q != SP::N_Q || D->n_qd != SP::N_QD || D->floating != SP::FLOATING) return false;
    if (E->n_act != 0) {
      if (E->n_act != SP::N_ACT) return false;
      for (int a = 0; a < SP::N_ACT; ++a) if (E->act_link[a] != SP::ACT_LINK[a]) return false;
    }
    auto trunk_q = [](int q) { const int k = k_of_q<SP, 0>(q); return k >= 0 && k < SP::N_TRUNK; };
    if (E->reward_kind == 1 && (SP::FLOATING || !trunk_q(0) || !trunk_q(2) || !trunk_q(3) || !trunk_q(4))) return false;
    if (E->reward_kind == 2 && !SP::FLOATING) return false;
    if (E->reward_kind == 3 && (SP::FLOATING || !trunk_q(0) || !trunk_q(2))) return false;
    return true;
  }
  // the dynamic part of the caller's flat model (everything but the visuals) must equal the compiled one bit for bit
  static bool same_model(const double* model, int n_model, const double* mine, int n_mine) {
    const int n_dyn = TDSM_HEADER + TDSM_BASE + SP::N_LINKS * TDSM_LINK + SP::N_GEOMS * TDSM_GEOM;
    if (n_dyn > n_mine || n_dyn > n_model) return false;
    for (int i = 0; i < n_dyn; ++i) {
      if (i == TDSM_H_NVIS) continue;
      if (!(model[i] == mine[i])) return false;
    }
    return true;
  }
  static size_t smem_bytes(int precision) {
    if (precision == 0) return (size_t)Lay<SP, float, double, float>::TOTAL * 32 * 4;
    if (precision == 1) return (size_t)Lay<SP, double, double, double>::TOTAL * 32 * 4;
    return (size_t)Lay<SP, float, float, float>::TOTAL * 32 * 4;
  }
  static int launch(const SimParams* P, const EnvParams* E, const StepIO* io, int mode, int use_pd, int precision, cudaStream_t stream) {
    const int tiles = (io->n + 31) / 32;
    const size_t smem1 = smem_bytes(precision);
    cudaError_t err = cudaSuccess;
    int dev_ = 0; cudaGetDevice(&dev_);
    static int sm_count[64] = {0};
    if (!sm_count[dev_ & 63]) cudaDeviceGetAttribute(&sm_count[dev_ & 63], cudaDevAttrMultiProcessorCount, dev_);
    static int smem_per_sm[64] = {0};
    if (!smem_per_sm[dev_ & 63]) cudaDeviceGetAttribute(&smem_per_sm[dev_ & 63], cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev_);
    // throughput mode: more tiles than two waves of single-tile CTAs and two tiles fit one CTA's shared memory
    static const int tpc_env = getenv("TDS_B200_TPC") ? atoi(getenv("TDS_B200_TPC")) : 0;
    // (opt-in until measured on the target: TDS_B200_TPC=2; TDS_B200_TPC=-1 = automatic for batches of more than two waves)
    int tpc = 1;
    if (tpc_env == -1) tpc = (tiles > 2 * sm_count[dev_ & 63] && 2 * smem1 <= 227 * 1024) ? 2 : 1;
    if (tpc_env == 2) tpc = 2 * smem1 <= 227 * 1024 ? 2 : 1;
    // Every step is a programmatic dependent launch: its grid may be scheduled before the previous kernel of the stream
    // (or the previous kernel node of a captured graph) has completed; the kernel does its step-independent prologue
    // and waits in griddepcontrol.wait for that kernel's completion and memory flush.  After a kernel that never
    // triggers (a policy kernel, the reset kernels, a kernel of another library) the dependency resolves when its
    // CTAs exit, as without the attribute.
    // When the grid is one wave (the tiles fit the device's co-resident CTA slots), the kernel triggers at entry (mode
    // bit 512): the next step's grid is scheduled while this one runs, and its CTAs take the SMs this one leaves idle and
    // each SM as soon as this step's CTA there exits, so only the wait separates the two steps.  This cannot starve the
    // running grid: a dependent grid is scheduled only after EVERY CTA of its primary has triggered or exited, i.e. when
    // all of the primary's CTAs are already resident, so a dependent CTA never holds a slot that the primary still needs.
    // Larger batches trigger after the tile's last store.
    // A grid of at most one CTA per SM asks for more than half of the SM's shared memory (smem_one), so that the
    // scheduler cannot put two of them on one SM.  Measured on the H100 (scripts/step_gaps.py, DESIGN.md section 4.3):
    // with two slots per SM, the next step's CTAs were placed next to running tiles, and the grid's span grew by as much
    // as the overlap saved.
#define TDSS_LAUNCH(RA, RC, RS, VAR, TPC)                                                               \
  do {                                                                                                  \
    auto k = tds_step_spec_kernel<SP, RA, RC, RS, VAR, TPC>;                                            \
    const size_t smem = smem1 * TPC;                                                                    \
    static bool attr_set_dev[64] = {false}; bool& attr_set = attr_set_dev[dev_ & 63]; /* the attribute is per device */ \
    static int ctas_per_sm_dev[64] = {0}; int& ctas_per_sm = ctas_per_sm_dev[dev_ & 63];              \
    const size_t smem_one = smem > (size_t)smem_per_sm[dev_ & 63] / 2 ? smem : (size_t)smem_per_sm[dev_ & 63] / 2; \
    if (!attr_set && smem_one > 48 * 1024) {                                                            \
      err = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_one);        \
      /* two tiles per SM when the batch has more tiles than SMs: ask for the largest shared-memory carveout */ \
      if (err == cudaSuccess) err = cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared); \
      if (err == cudaSuccess) attr_set = true;                                                          \
    }                                                                                                   \
    if (err == cudaSuccess && !ctas_per_sm)                                                             \
      err = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas_per_sm, k, 32 * TDS_TEAM_T * TPC, smem); \
    if (err == cudaSuccess) {                                                                           \
      const int ctas = (tiles + TPC - 1) / TPC;                                                         \
      const bool one_per_sm = ctas <= sm_count[dev_ & 63];                                              \
      cudaLaunchConfig_t cfg = {};                                                                      \
      cfg.gridDim = dim3(ctas); cfg.blockDim = dim3(32 * TDS_TEAM_T * TPC);                             \
      cfg.dynamicSmemBytes = one_per_sm ? smem_one : smem; cfg.stream = stream;                         \
      cudaLaunchAttribute at[1];                                                                        \
      at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;                                    \
      at[0].val.programmaticStreamSerializationAllowed = 1;                                             \
      cfg.attrs = at; cfg.numAttrs = 1;                                                                 \
      const int mode_k = mode | (one_per_sm || ctas <= ctas_per_sm * sm_count[dev_ & 63] ? 512 : 0);   \
      err = cudaLaunchKernelEx(&cfg, k, *P, *E, *io, mode_k, use_pd);                                   \
    }                                                                                                   \
  } while (0)
    // instance: general (extra outputs / forward dynamics only), lean, lean + host layouts
    const int var = ((mode & 255) == 0 || io->link_xf || io->contact_dist || io->qdd_out) ? 0 : ((io->act_aos && use_pd) ? 2 : 1);
    if (var != 2 && io->act_aos) return (int)cudaErrorInvalidValue;   // host layouts are only served by the lean instance
#define TDSS_PREC(VAR, TPC)                                                      \
  do {                                                                           \
    if (precision == 0) TDSS_LAUNCH(float, double, float, VAR, TPC);             \
    else if (precision == 1) TDSS_LAUNCH(double, double, double, VAR, TPC);      \
    else TDSS_LAUNCH(float, float, float, VAR, TPC);                             \
  } while (0)
    if (var == 0) TDSS_PREC(0, 1);
#ifdef TDS_B200_WITH_TPC2   // measured slower than independent CTAs: compiled on request only
    else if (var == 1 && tpc == 2 && precision != 1) { if (precision == 0) TDSS_LAUNCH(float, double, float, 1, 2); else TDSS_LAUNCH(float, float, float, 1, 2); }
    else if (var == 2 && tpc == 2 && precision != 1) { if (precision == 0) TDSS_LAUNCH(float, double, float, 2, 2); else TDSS_LAUNCH(float, float, float, 2, 2); }
#endif
    else if (var == 1) TDSS_PREC(1, 1);
    else TDSS_PREC(2, 1);
#undef TDSS_PREC
#undef TDSS_LAUNCH
    return (int)err;
  }
};
#endif  // TDS_STEPS_KERNEL_ONLY

}  // namespace tdss

// ---- the models compiled into this library -----------------------------------------------------------------------------
// per-role / trunk constant tables + table accessors of one spec
#define TDS_SPEC_TABLES(SP, sym)                                                                                          \
  namespace tdss {                                                                                                        \
  __constant__ LegTab<SP> c_legs_##sym[TDS_TEAM_T] = {make_leg<SP>(0), make_leg<SP>(1), make_leg<SP>(2), make_leg<SP>(3)}; \
  template <> __device__ __forceinline__ const LegTab<SP>& leg_tab<SP>(int role) { return c_legs_##sym[role]; }            \
  __constant__ TrunkTab<SP> c_trunk_##sym = make_trunk<SP>();                                                             \
  template <> __device__ __forceinline__ const TrunkTab<SP>& trunk_tab<SP>() { return c_trunk_##sym; }                    \
  __constant__ CandTab<SP> c_cand_##sym = make_cand<SP>();                                                                \
  template <> __device__ __forceinline__ const CandTab<SP>& cand_tab<SP>() { return c_cand_##sym; }                       \
  }
TDS_SPEC_TABLES(SpecLaikago, laikago)
TDS_SPEC_TABLES(SpecAnt, ant)

#ifndef TDS_STEPS_KERNEL_ONLY
static const double k_spec_laikago_model[] = {
#include "generated/laikago_model.inc"
};
static const double k_spec_ant_model[] = {
#include "generated/ant_model.inc"
};

// Which ahead-of-time compiled kernel covers this simulator?  (same flat model, bit for bit, and same actuator map)
// Returns the spec index (0 Laikago, 1 Ant) or -1.
extern "C" int tds_spec_find(const double* model, int n_model, const DevModel* D, const EnvParams* E) {
  using namespace tdss;
  if (SpecHost<SpecLaikago>::same_model(model, n_model, k_spec_laikago_model, (int)(sizeof(k_spec_laikago_model) / sizeof(double))) &&
      SpecHost<SpecLaikago>::matches(D, E)) return 0;
  if (SpecHost<SpecAnt>::same_model(model, n_model, k_spec_ant_model, (int)(sizeof(k_spec_ant_model) / sizeof(double))) &&
      SpecHost<SpecAnt>::matches(D, E)) return 1;
  return -1;
}

extern "C" size_t tds_spec_smem_bytes(int spec, int precision) {
  using namespace tdss;
  return spec == 0 ? SpecHost<SpecLaikago>::smem_bytes(precision) : SpecHost<SpecAnt>::smem_bytes(precision);
}

extern "C" const char* tds_spec_name(int spec) { return spec == 0 ? "laikago" : (spec == 1 ? "ant" : ""); }

extern "C" int tds_launch_step_spec(int spec, const SimParams* P, const EnvParams* E, const StepIO* io, int mode, int use_pd,
                                    int precision, cudaStream_t stream) {
  using namespace tdss;
  if (spec == 0) return SpecHost<SpecLaikago>::launch(P, E, io, mode, use_pd, precision, stream);
  if (spec == 1) return SpecHost<SpecAnt>::launch(P, E, io, mode, use_pd, precision, stream);
  return (int)cudaErrorInvalidValue;
}
#endif  // TDS_STEPS_KERNEL_ONLY
