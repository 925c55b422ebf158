// Step body of the two table-driven tree kernels: the lane-team kernel (tds_stept.cu) and the role-warp kernel
// (tds_stepr.cu).  The algorithm is written once here; each kernel's file only says how threads are mapped.
//
// With 4096 environments a one-lane-per-environment kernel leaves every SM with a single warp whose
// instruction stream is paid at full latency (tds_stepw.cu: ~160k cycles per step).  The serial length per
// environment is what bounds the step, so the work of ONE environment is cut along the kinematic tree
// (host side: tds_team.h) into TDS_TEAM_T = 4 roles: role 0 owns the TRUNK (root chain up to the branching
// links) plus one subtree, roles 1..3 own one subtree each (Laikago: 6 trunk links + one leg per role).
// Everything is expressed in the common world-aligned frame of tds_stepw.cu, so subtree results combine by
// plain sums:
//   * pass 1 / pass 3 (root -> leaf): role 0 walks the trunk, publishes the attachment transforms /
//     accelerations in the shared region of the environment, then all roles walk their subtree;
//   * pass 2 (leaf -> root): every role reduces its subtree into attachment accumulators (articulated inertia,
//     bias force, composite inertia); the four partial accumulators are summed; role 0 finishes the trunk;
//   * M is never assembled: leaf-first block elimination.  Per role: own block M_kk = L_k L_k^T,
//     G_k = L_k^-1 C_k (coupling with the trunk dofs); Schur complement S = B - sum_k G_k^T G_k =
//     L_t L_t^T on role 0.  A contact row touches only its owner's dofs and the trunk dofs, so
//     Y = L^-1 Jc^T is computed by the owning role alone;
//   * projected Gauss-Seidel keeps the reference's row order (normals | friction 1 | friction 2, contacts in
//     enumeration order); w = Y p is split into a private part and the shared trunk part, which the owner of
//     a row updates in place and a barrier publishes before a row of another owner reads it.
// Scalar types as in tds_stepw.cu (RA fp32 ABA, RC fp64 kinematics/inertias/CRBA products/Jacobians/rhs,
// RS fp32 factorisation + PGS).  Reference citations are given at each stage.
//
// The policy `Map` places the four roles of an environment on threads.  A tile is the set of STM environments
// that share one block of scratch: the shared region [word][environment] (coordinates, trunk records, trunk
// factor), then the role-private regions [word][lane].
//   * LaneTeam (tds_stept.cu): four adjacent lanes per environment, a tile is the 8 environments of a one-warp
//     CTA.  The link table is read from global memory through the non-coherent path.  Roles meet at
//     __syncwarp; sums over the roles are a shuffle butterfly (v + shfl 1) + shfl 2 that every lane receives.
//   * RoleWarps (tds_stepr.cu): role = warp of a 128-thread CTA, lane = environment, a tile is the CTA's 32
//     environments.  Every lane of a warp runs the same link, so the link table sits in constant memory.
//     Roles meet at CTA barriers; role 0 sums the partial results (p0 + p1) + (p2 + p3) of the other roles
//     from their private regions.
// The two sums round differently, so the kernels agree with each other to rounding, not bit for bit.
// A policy holds: THREADS, MIN_BLOCKS (launch bounds), STM, ROLE_WARPS (selects the reductions, barriers and
// PGS row loop below), MAX_CARVEOUT (launch), and role(), team(), tile(), table(), ld(), sync(), tile_bytes(),
// role_base(), clock_row().
#pragma once
#include <cuda_runtime.h>

#include "tds_wcommon.cuh"
#include "tds_team.h"

namespace tdsteam {
using namespace tds;
using namespace tdsw;

constexpr int TT = TDS_TEAM_T;         // roles per environment
constexpr int SL = 32;                 // element stride of a role-private region: [word][lane]

// sum over a lane team; every lane receives the same bits (commutative pairwise tree)
template <typename T> TDS_D T team_sum(T v, unsigned mask) {
  v += __shfl_xor_sync(mask, v, 1);
  v += __shfl_xor_sync(mask, v, 2);
  return v;
}

template <class Map, typename RA, typename RC, typename RS, bool SMEM>
__global__ void __launch_bounds__(Map::THREADS, Map::MIN_BLOCKS)
tds_team_step_kernel(const __grid_constant__ TeamModel TM, const TeamLink* __restrict__ tl,
                     const __grid_constant__ DevModel M, const __grid_constant__ SimParams P,
                     const __grid_constant__ EnvParams E, const StepIO io, const int mode, const int use_pd,
                     char* __restrict__ gscratch) {
  constexpr int STM = Map::STM;          // element stride of the shared region: environments per tile
  extern __shared__ __align__(16) char smem_raw[];
  const int lane = threadIdx.x & 31;
  const int role = Map::role();
  const int team = Map::team();          // column of this environment in the shared region
  const int tile = Map::tile();
  const int env = tile * STM + team;
  const bool live = env < io.n;
  const int e = live ? env : io.n - 1;
  const unsigned tmask = 0xFu << (team * TT);   // LaneTeam: the lanes of this environment
  // SMEM is a template parameter so that the compiler keeps the shared address space (LDS/STS, 32-bit addressing)
  char* const tb = SMEM ? smem_raw : gscratch + (size_t)tile * Map::tile_bytes(TM);
  char* const lb = Map::role_base(TM, tb, role);
  auto tp = [&](int word, auto tag) { using T = decltype(tag); return (sizeof(T) == 4) ? ((T*)tb) + (size_t)word * STM + team : ((T*)tb) + (size_t)(word >> 1) * STM + team; };
  auto lp = [&](int word, auto tag) { using T = decltype(tag); return (sizeof(T) == 4) ? ((T*)lb) + (size_t)word * SL + lane : ((T*)lb) + (size_t)(word >> 1) * SL + lane; };
  const int ns = io.n_stride;
  const int n_trunk = TM.n_trunk, n_td = TM.n_td, nbt = TM.nbt, nt3 = 3 * TM.nbt;
  const int n_loc = TM.n_loc[role], n_od = TM.n_od[role], nbo = TM.nbo[role];
  const TeamLink* const mytl = Map::table(tl, role);
  constexpr int RAW = (int)(sizeof(RA) / 4), RCW = (int)(sizeof(RC) / 4);
  const int LWD = TM.link_words, UOFF = 10 * RCW, VOFF = 10 * RCW + 8 * RAW;
  int phase_id = 0;
#define TDST_PHASE() do { if (io.phase_clk && lane == 0) io.phase_clk[Map::clock_row(tile, role) * 16 + phase_id] = clock64(); ++phase_id; } while (0)
  TDST_PHASE();

#ifndef TDS_TEAM_KERNEL_ONLY   // (the host-compiled copy of the kernel source in tests/cpp has no PTX)
  if constexpr (!Map::ROLE_WARPS) {
    // warm L1 with the per-role link tables (read many times below through the non-coherent path) and issue the
    // loads of this team's coordinates early; a lone warp otherwise pays one L2 round trip per first touch
    const char* tbl = (const char*)tl;
    const int lines = (TDS_TEAM_T * TDS_TEAM_MAXK * (int)sizeof(TeamLink) + 127) / 128;
    for (int l = lane; l < lines; l += 32) asm volatile("prefetch.global.L1 [%0];" ::"l"(tbl + (size_t)l * 128));
  }
#endif

  float* const tq = tp(TM.t_q, 0.f);
  float* const tqd = tp(TM.t_qd, 0.f);
  float* const ttau = tp(TM.t_tau, 0.f);
  // coordinate accessors of a local link: all coordinates of the environment live in the shared region at their
  // global index
  auto q_ref = [&](const int, const int q_idx, const int) -> float& { return tq[q_idx * STM]; };
  auto qd_ref = [&](const int, const int qd_idx, const int) -> float& { return tqd[qd_idx * STM]; };
  auto tau_ref = [&](const int, const int qd_idx, const int) -> float& { return ttau[qd_idx * STM]; };

  // ---- load state (the four roles share the rows, all loads independent -> one memory round trip),
  //      PD torques (locomotion_contact_simulation.h:168-258) ---------------------------------------------
  const int k_first = (role == 0) ? 0 : n_trunk;     // role 0 also owns the trunk
#pragma unroll 4
  for (int k = role; k < M.n_q; k += TT) tq[k * STM] = io.q_in[(size_t)k * ns + e];
#pragma unroll 4
  for (int k = role; k < M.n_qd; k += TT) { tqd[k * STM] = io.qd_in[(size_t)k * ns + e]; ttau[k * STM] = 0.f; }
  Map::sync();
  if (use_pd) {
#pragma unroll 4
    for (int a = role; a < E.n_act; a += TT) {
      const int li = E.act_link[a];
      float act = io.tau_in[(size_t)a * ns + e];
      act = fmaxf(fminf(act, E.action_limit), -E.action_limit);
      const float q_des = E.initial_poses[a] + act;
      const float f = E.kp * (q_des - tq[M.q_idx[li] * STM]) + E.kd * (0.f - tqd[M.qd_idx[li] * STM]);
      ttau[M.qd_idx[li] * STM] = fminf(fmaxf(f, -E.max_force), E.max_force);
    }
  } else if (io.tau_in) {
    const int off = M.floating ? 6 : 0;
#pragma unroll 4
    for (int k = off + role; k < M.n_qd; k += TT) ttau[k * STM] = io.tau_in[(size_t)(k - off) * ns + e];
  }
  for (int s = 0; s < TM.n_acc; ++s) {
    RA* pa = lp(TM.l_acc + s * TM.acc_words, RA(0));
    for (int k = 0; k < 27; ++k) pa[k * SL] = RA(0);
    RC* pc = lp(TM.l_acc + s * TM.acc_words + TM.acc_ic_word, RC(0));
    for (int k = 0; k < 10; ++k) pc[k * SL] = RC(0);
  }
  const bool want_contacts = (mode == MODE_FULL) && M.has_plane;
  const V3<RC> pn = v3<RC>(RC(M.plane_n[0]), RC(M.plane_n[1]), RC(M.plane_n[2]));
  RC* const tO = tp(TM.t_O, RC(0));     // O[3], plane_off, Rb[9]
  // RoleWarps: the XTRA words behind the shared region, active masks [2 * role + {lo, hi}] then the done flag
  unsigned* const amask = (unsigned*)tb + (size_t)TM.t_total * STM + lane;
  Map::sync();
  TDST_PHASE();  // 1

  // ---- contact candidates of this role ----------------------------------------------------------------------
  unsigned long long my_active = 0ull;   // bit = global candidate index
  int n_my_active = 0;
  auto emit_geoms = [&](const int g_begin, const int g_end, int cand, int lpt, const int link_local, const M3<RC>& R,
                        const V3<RC>& pr, const RC plane_off) {
    for (int g = g_begin; g < g_end; ++g) {
      const int ty = M.g_type[g];
      if (ty != TDSG_SPHERE && ty != TDSG_CAPSULE) continue;
      const V3<RC> c = pr + mul(R, v3<RC>(RC(M.g_t[g][0]), RC(M.g_t[g][1]), RC(M.g_t[g][2])));
      const RC rad = RC(M.g_radius[g]);
      const int npts = (ty == TDSG_CAPSULE) ? 2 : 1;
      V3<RC> half = v3<RC>(RC(0), RC(0), RC(0));
      if (ty == TDSG_CAPSULE) half = mul(R, v3<RC>(RC(M.g_half[g][0]), RC(M.g_half[g][1]), RC(M.g_half[g][2])));
      for (int k = 0; k < npts; ++k) {
        const V3<RC> pos = (ty == TDSG_CAPSULE) ? (k == 0 ? c + half : c - half) : c;
        const RC dist = dot(pos, pn) + plane_off - rad;       // contact_point.hpp:112-116
        if (io.contact_dist && live) io.contact_dist[(size_t)cand * ns + e] = (float)dist;
        RC* pc = lp(TM.l_con + lpt * 5 * RCW, RC(0));
        pc[4 * SL] = RC(-100);                                  // inactive marker
        if (dist < RC(0)) {
          st3<RC>(pc, SL, pos - pn * rad);                     // world_point_on_b, relative to O
          pc[3 * SL] = dist;
          pc[4 * SL] = RC(link_local);
          my_active |= 1ull << cand;
          ++n_my_active;
        }
        ++cand; ++lpt;
      }
    }
  };

  // ---- pass 1 on one link (kinematics.hpp:18-148, link.hpp:229-336) in the common frame ------------------------
  // carried state
  M3<RC> R_prev; V3<RC> p_prev; Sv<RA> v_prev;
  auto pass1_link = [&](const int k, RC* const Srec, char* const rec_rc /*RC view*/, char* const rec_ra /*RA view*/,
                        const int ST, const RC plane_off, const V3<RC>& O) {
    const TeamLink& L = mytl[k];
    const int fl = Map::ld(L.flags);
    const int lpar = Map::ld(L.lpar);
    M3<RC> Rp; V3<RC> pp; Sv<RA> vp;
    if (fl & TDS_TF_PARENT_ADJ) { Rp = R_prev; pp = p_prev; vp = v_prev; }
    else if (lpar < 0) {            // base
      const RC* px = tp(TM.t_xw, RC(0));
      Rp = ld9<RC>(px, STM); pp = ld3<RC>(px + 9 * STM, STM);
      vp = ld6<RA>(tp(TM.t_xw + 12 * RCW * (TM.n_xw_team + 1), RA(0)), STM);   // base velocity (see below)
    } else if (lpar < n_trunk) {    // trunk parent: published by role 0 in the shared region
      const int xs = Map::ld(mytl[lpar].xw_slot);
      const RC* px = tp(TM.t_xw + (xs + 1) * 12 * RCW, RC(0));
      Rp = ld9<RC>(px, STM); pp = ld3<RC>(px + 9 * STM, STM);
      vp = ld6<RA>(tp(TM.t_link + lpar * LWD + VOFF, RA(0)), STM);
    } else {                        // own branch parent
      const int xs = Map::ld(mytl[lpar].xw_slot);
      const RC* px = lp(TM.l_xw + xs * 12 * RCW, RC(0));
      Rp = ld9<RC>(px, SL); pp = ld3<RC>(px + 9 * SL, SL);
      vp = ld6<RA>(lp(TM.l_link + (lpar - n_trunk) * LWD + VOFF, RA(0)), SL);
    }
    V3<RC> pi = pp + mul(Rp, v3<RC>(RC(Map::ld(L.XT[9])), RC(Map::ld(L.XT[10])), RC(Map::ld(L.XT[11]))));
    M3<RC> Ri = Rp;
    if (!(fl & TDS_LF_XT_IDENT)) {
      M3<RC> r; r.xx = RC(Map::ld(L.XT[0])); r.xy = RC(Map::ld(L.XT[1])); r.xz = RC(Map::ld(L.XT[2])); r.yx = RC(Map::ld(L.XT[3])); r.yy = RC(Map::ld(L.XT[4])); r.yz = RC(Map::ld(L.XT[5])); r.zx = RC(Map::ld(L.XT[6])); r.zy = RC(Map::ld(L.XT[7])); r.zz = RC(Map::ld(L.XT[8]));
      Ri = mul(Rp, r);
    }
    Sv<RC> S; S.top = v3<RC>(RC(0), RC(0), RC(0)); S.bot = S.top;
    const int qi_ = Map::ld(L.q_idx), qdi_ = Map::ld(L.qd_idx), ld_ = Map::ld(L.ldof);
    if (!(fl & TDS_LF_FIXED)) {
      const RC qi = RC(q_ref(k, qi_, ld_));
      const int jt = Map::ld(L.jtype);
      const V3<RC> ax = v3<RC>(RC(Map::ld(L.axis[0])), RC(Map::ld(L.axis[1])), RC(Map::ld(L.axis[2])));
      if (fl & TDS_LF_PRISMATIC) {
        const V3<RC> d = mul(Ri, ax);
        pi = axpy(d, qi, pi);
        S.bot = d;
      } else {
        const V3<RC> w = mul(Ri, ax);
        if (jt == TDSJ_REVOLUTE_AXIS) {
          const RC dl = sqrt_t(dot(ax, ax));
          RC s, c;
          sincos_t(qi * RC(0.5), &s, &c);
          s = s / dl;
          Ri = mul(Ri, quat_to_matrix<RC>(ax.x * s, ax.y * s, ax.z * s, c));
        } else {
          RC s, c;
          sincos_t(qi, &s, &c);
          const V3<RC> cx = col_x(Ri), cy = col_y(Ri), cz = col_z(Ri);
          if (jt == TDSJ_REVOLUTE_X) set_cols(Ri, cx, axpy(cz, s, cy * c), axpy(cy, -s, cz * c));
          else if (jt == TDSJ_REVOLUTE_Y) set_cols(Ri, axpy(cz, -s, cx * c), cy, axpy(cx, s, cz * c));
          else set_cols(Ri, axpy(cy, s, cx * c), axpy(cx, -s, cy * c), cz);
        }
        S.top = w;
        S.bot = cross(pi, w);
      }
    }
    st6<RC>(Srec, ST, S);
    const int xs = Map::ld(L.xw_slot);
    if (xs >= 0) {
      if (k < n_trunk) { RC* px = tp(TM.t_xw + (xs + 1) * 12 * RCW, RC(0)); st9<RC>(px, STM, Ri); st3<RC>(px + 9 * STM, STM, pi); }
      else { RC* px = lp(TM.l_xw + xs * 12 * RCW, RC(0)); st9<RC>(px, SL, Ri); st3<RC>(px + 9 * SL, SL, pi); }
    }
    {   // rigid-body inertia about O in world axes
      Rbi<RC> r;
      r.m = RC(Map::ld(L.rbic[0]));
      const V3<RC> c = pi + mul(Ri, v3<RC>(RC(Map::ld(L.rbic[1])), RC(Map::ld(L.rbic[2])), RC(Map::ld(L.rbic[3]))));
      r.h = c * r.m;
      S3<RA> Icf; Icf.xx = RA(Map::ld(L.rbic[4])); Icf.xy = RA(Map::ld(L.rbic[5])); Icf.xz = RA(Map::ld(L.rbic[6])); Icf.yy = RA(Map::ld(L.rbic[7])); Icf.yz = RA(Map::ld(L.rbic[8])); Icf.zz = RA(Map::ld(L.rbic[9]));
      const S3<RA> Irot = rot_sym(cvt<RA>(Ri), Icf);
      r.I.xx = RC(Irot.xx); r.I.xy = RC(Irot.xy); r.I.xz = RC(Irot.xz); r.I.yy = RC(Irot.yy); r.I.yz = RC(Irot.yz); r.I.zz = RC(Irot.zz);
      const RC cc = dot(c, c);
      r.I.xx += r.m * (cc - c.x * c.x); r.I.yy += r.m * (cc - c.y * c.y); r.I.zz += r.m * (cc - c.z * c.z);
      r.I.xy -= r.m * c.x * c.y; r.I.xz -= r.m * c.x * c.z; r.I.yz -= r.m * c.y * c.z;
      st_rbi<RC>((RC*)rec_rc, ST, r);
    }
    Sv<RA> v = vp;
    if (!(fl & TDS_LF_FIXED)) {
      const RA qdi = RA(qd_ref(k, qdi_, ld_));
      const Sv<RA> Sf = cvt_sv<RA>(S);
      v.top = axpy(Sf.top, qdi, v.top);
      v.bot = axpy(Sf.bot, qdi, v.bot);
    }
    st6<RA>((RA*)rec_ra, ST, v);
    if (want_contacts) emit_geoms(Map::ld(L.g_begin), Map::ld(L.g_end), Map::ld(L.cand_begin), Map::ld(L.lpt_begin), k, Ri, pi, plane_off);
    if (io.link_xf && live) {
      float* o = io.link_xf + (size_t)Map::ld(L.link) * 12 * ns + e;
      o[0] = (float)Ri.xx; o[(size_t)1 * ns] = (float)Ri.xy; o[(size_t)2 * ns] = (float)Ri.xz;
      o[(size_t)3 * ns] = (float)Ri.yx; o[(size_t)4 * ns] = (float)Ri.yy; o[(size_t)5 * ns] = (float)Ri.yz;
      o[(size_t)6 * ns] = (float)Ri.zx; o[(size_t)7 * ns] = (float)Ri.zy; o[(size_t)8 * ns] = (float)Ri.zz;
      o[(size_t)9 * ns] = (float)(pi.x + O.x); o[(size_t)10 * ns] = (float)(pi.y + O.y); o[(size_t)11 * ns] = (float)(pi.z + O.z);
    }
    R_prev = Ri; p_prev = pi; v_prev = v;
  };
  auto trunk_rec = [&](int k, int off, auto tag) { return tp(TM.t_link + k * LWD + off, tag); };
  auto own_rec = [&](int k, int off, auto tag) { return lp(TM.l_link + (k - n_trunk) * LWD + off, tag); };

  // ---- pass 1a: role 0 computes the origin and walks the trunk ------------------------------------------------
  RA* const tvbase = tp(TM.t_xw + 12 * RCW * (TM.n_xw_team + 1), RA(0));   // base velocity (6 RA) behind the xw slots
  if (role == 0) {
    M3<RC> Rb = m3_identity<RC>();
    V3<RC> O = v3<RC>(RC(0), RC(0), RC(0));
    if (M.floating) {
      Rb = quat_to_matrix<RC>(RC(tq[0]), RC(tq[STM]), RC(tq[2 * STM]), RC(tq[3 * STM]));
      O = v3<RC>(RC(tq[4 * STM]), RC(tq[5 * STM]), RC(tq[6 * STM]));
    } else {   // end of the translation-only root chain (links 0..n_prefix-1 are trunk links of a chain)
      M3<RC> Rc = m3_identity<RC>();
      const int kp = M.n_prefix < M.n_links ? M.n_prefix + 1 : M.n_links;
      for (int i = 0; i < kp; ++i) {
        const double* xt = M.XT[i];
        O = O + mul(Rc, v3<RC>(RC(xt[9]), RC(xt[10]), RC(xt[11])));
        if (i == M.n_prefix) break;
        if (!(M.flags[i] & TDS_LF_XT_IDENT)) {
          M3<RC> r; r.xx = RC(xt[0]); r.xy = RC(xt[1]); r.xz = RC(xt[2]); r.yx = RC(xt[3]); r.yy = RC(xt[4]); r.yz = RC(xt[5]); r.zx = RC(xt[6]); r.zy = RC(xt[7]); r.zz = RC(xt[8]);
          Rc = mul(Rc, r);
        }
        if (M.flags[i] & TDS_LF_PRISMATIC) {
          const RC qi = RC(io.q_in[(size_t)M.q_idx[i] * ns + e]);
          O = O + mul(Rc, v3<RC>(RC(M.axis[i][0]) * qi, RC(M.axis[i][1]) * qi, RC(M.axis[i][2]) * qi));
        }
      }
    }
    const RC plane_off = dot(O, pn) - RC(M.plane_c);
    st3<RC>(tO, STM, O); tO[3 * STM] = plane_off; st9<RC>(tO + 4 * STM, STM, Rb);
    R_prev = Rb;
    p_prev = M.floating ? v3<RC>(RC(0), RC(0), RC(0)) : v3<RC>(-O.x, -O.y, -O.z);
    if (M.floating) {
      const M3<RA> RbA = cvt<RA>(Rb);
      v_prev.top = mul(RbA, v3<RA>(RA(tqd[0]), RA(tqd[STM]), RA(tqd[2 * STM])));
      v_prev.bot = mul(RbA, v3<RA>(RA(tqd[3 * STM]), RA(tqd[4 * STM]), RA(tqd[5 * STM])));
    } else { v_prev.top = v3<RA>(RA(0), RA(0), RA(0)); v_prev.bot = v_prev.top; }
    { RC* px = tp(TM.t_xw, RC(0)); st9<RC>(px, STM, R_prev); st3<RC>(px + 9 * STM, STM, p_prev); }
    st6<RA>(tvbase, STM, v_prev);
    if (want_contacts) emit_geoms(M.geom_begin[0], M.geom_begin[1], 0, 0, -1, R_prev, p_prev, plane_off);
    for (int k = 0; k < n_trunk; ++k)
      pass1_link(k, tp(TM.t_S + k * 6 * RCW, RC(0)), (char*)trunk_rec(k, 0, RC(0)), (char*)trunk_rec(k, VOFF, RA(0)), STM, plane_off, O);
  }
  Map::sync();
  // ---- pass 1b: every role walks its subtree ------------------------------------------------------------------------
  const V3<RC> O = ld3<RC>(tO, STM);
  const RC plane_off = tO[3 * STM];
  const M3<RC> Rb = ld9<RC>(tO + 4 * STM, STM);
  for (int k = n_trunk; k < n_loc; ++k)
    pass1_link(k, lp(TM.l_S + (k - n_trunk) * 6 * RCW, RC(0)), (char*)own_rec(k, 0, RC(0)), (char*)own_rec(k, VOFF, RA(0)), SL, plane_off, O);
  // set of active candidates of the environment (OR over the roles), and whether any of the environments whose
  // threads meet at the barriers of the contact solve has one: those threads enter or skip the solve together
  unsigned long long team_active;
  bool any_contact;
  if constexpr (Map::ROLE_WARPS) {   // through the shared region; any contact in the tile
    amask[(2 * role) * STM] = (unsigned)my_active;
    amask[(2 * role + 1) * STM] = (unsigned)(my_active >> 32);
    any_contact = __syncthreads_or(my_active != 0ull) != 0;
    team_active = 0ull;
#pragma unroll
    for (int r = 0; r < TT; ++r) team_active |= ((unsigned long long)amask[(2 * r + 1) * STM] << 32) | amask[(2 * r) * STM];
  } else {   // xor shuffles over the team; any contact of this environment
    unsigned lo = (unsigned)my_active, hi = (unsigned)(my_active >> 32);
    lo |= __shfl_xor_sync(tmask, lo, 1); lo |= __shfl_xor_sync(tmask, lo, 2);
    hi |= __shfl_xor_sync(tmask, hi, 1); hi |= __shfl_xor_sync(tmask, hi, 2);
    team_active = ((unsigned long long)hi << 32) | lo;
    any_contact = team_active != 0ull;
  }
  const bool team_contact = team_active != 0ull;
  TDST_PHASE();  // 2

  // ---- pass 2 on one link: ABA (forward_dynamics.hpp:50-216) + CRBA (mass_matrix.hpp:39-125) ------------------
  RS* const Mkk = lp(TM.l_M, RS(0));
  RS* const Ck = lp(TM.l_C, RS(0));         // block (bo, bt) at ((bo * nbt + bt) * 9)
  RS* const Bt = tp(TM.t_B, RS(0));
  Abi<RA> cA; Sv<RA> cP; Rbi<RC> cC;
  auto S_of = [&](int k) -> Sv<RC> { return k < n_trunk ? ld6<RC>(tp(TM.t_S + k * 6 * RCW, RC(0)), STM) : ld6<RC>(lp(TM.l_S + (k - n_trunk) * 6 * RCW, RC(0)), SL); };
  auto pass2_link = [&](const int k, char* const rec0, char* const recv, const int ST) {
    const TeamLink& L = mytl[k];
    const int fl = Map::ld(L.flags);
    RC* const rec = (RC*)rec0;
    RA* const vrec = (RA*)recv;
    Rbi<RC> Ic = ld_rbi<RC>(rec, ST);
    const Rbi<RA> rb = cvt_rbi<RA>(Ic);
    const Sv<RA> v = ld6<RA>(vrec, ST);
    Abi<RA> Ia = abi_from_rbi(rb);
    Sv<RA> pA = cross_mf(v, rbi_mul(rb, v));                 // kinematics.hpp:132
    if (fl & TDS_TF_CHILD_ADJ) { abi_add(Ia, cA); pA = pA + cP; rbi_add(Ic, cC); }
    const int as = Map::ld(L.acc_slot);
    if (as >= 0) {
      Abi<RA> sa; Sv<RA> sp;
      acc_ld27<RA>(lp(TM.l_acc + as * TM.acc_words, RA(0)), SL, sa, sp);
      abi_add(Ia, sa); pA = pA + sp;
      rbi_add(Ic, ld_rbi<RC>(lp(TM.l_acc + as * TM.acc_words + TM.acc_ic_word, RC(0)), SL));
    }
    Sv<RA> pa = pA;
    RA* const urec = (RA*)(k < n_trunk ? (char*)tp(TM.t_link + k * LWD + UOFF, RA(0)) : (char*)lp(TM.l_link + (k - n_trunk) * LWD + UOFF, RA(0)));
    if (fl & TDS_LF_FIXED) {
      Sv<RA> z; z.top = v3<RA>(RA(0), RA(0), RA(0)); z.bot = z.top;
      st6<RA>(vrec, ST, z);
      st6<RA>(urec, ST, z);
      urec[6 * ST] = RA(0); urec[7 * ST] = RA(0);
    } else {
      const Sv<RC> Sd = S_of(k);
      const Sv<RA> S = cvt_sv<RA>(Sd);
      const int qi_ = Map::ld(L.q_idx), qdi_ = Map::ld(L.qd_idx), ld_ = Map::ld(L.ldof);
      const RA qdj = RA(qd_ref(k, qdi_, ld_));
      Sv<RA> vJ; vJ.top = S.top * qdj; vJ.bot = S.bot * qdj;
      const Sv<RA> c = cross_mm(v, vJ);                      // kinematics.hpp:96-97
      const Sv<RA> U = abi_mul(Ia, S);                       // forward_dynamics.hpp:111
      const RA D = dot(S, U);
      const RA invD = RA(1) / D;
      RA tau = RA(tau_ref(k, qdi_, ld_));
      tau -= RA(Map::ld(L.stiffness)) * RA(q_ref(k, qi_, ld_));
      tau -= RA(Map::ld(L.damping)) * qdj;
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
      if (team_contact) {   // CRBA column (mass_matrix.hpp:86-111): M_ij = S_j . (Ic_i S_i)
        const Sv<RC> F = rbi_mul(Ic, Sd);
        const RS mii = RS(dot(Sd, F));
        if (k < n_trunk) {
          const int bi = ld_ / 3, ri = ld_ - 3 * bi;
          Bt[(btri(bi, bi) + ri * 4) * STM] = mii;
          for (int j = Map::ld(L.lpar); j >= 0; j = Map::ld(mytl[j].lpar)) {
            const int lj = Map::ld(mytl[j].ldof);
            if (lj < 0) continue;
            const int bj = lj / 3, cj = lj - 3 * bj;
            Bt[(btri(bi, bj) + ri * 3 + cj) * STM] = RS(dot(S_of(j), F));
          }
          if (M.floating) {
            const V3<RC> ft = mulT(Rb, F.top), fb = mulT(Rb, F.bot);
            RS* row0 = Bt + (btri(bi, 0) + ri * 3) * STM;
            RS* row1 = Bt + (btri(bi, 1) + ri * 3) * STM;
            row0[0] = RS(ft.x); row0[STM] = RS(ft.y); row0[2 * STM] = RS(ft.z);
            row1[0] = RS(fb.x); row1[STM] = RS(fb.y); row1[2 * STM] = RS(fb.z);
          }
        } else {
          const int oi = ld_ - n_td;
          const int bi = oi / 3, ri = oi - 3 * bi;
          Mkk[(btri(bi, bi) + ri * 4) * SL] = mii;
          for (int j = Map::ld(L.lpar); j >= 0; j = Map::ld(mytl[j].lpar)) {
            const int lj = Map::ld(mytl[j].ldof);
            if (lj < 0) continue;
            const RS val = RS(dot(S_of(j), F));
            if (lj >= n_td) { const int oj = lj - n_td, bj = oj / 3, cj = oj - 3 * bj; Mkk[(btri(bi, bj) + ri * 3 + cj) * SL] = val; }
            else { const int bj = lj / 3, cj = lj - 3 * bj; Ck[((bi * nbt + bj) * 9 + ri * 3 + cj) * SL] = val; }
          }
          if (M.floating) {
            const V3<RC> ft = mulT(Rb, F.top), fb = mulT(Rb, F.bot);
            RS* row0 = Ck + ((bi * nbt + 0) * 9 + ri * 3) * SL;
            RS* row1 = Ck + ((bi * nbt + 1) * 9 + ri * 3) * SL;
            row0[0] = RS(ft.x); row0[SL] = RS(ft.y); row0[2 * SL] = RS(ft.z);
            row1[0] = RS(fb.x); row1[SL] = RS(fb.y); row1[2 * SL] = RS(fb.z);
          }
        }
      }
    }
    if (fl & TDS_TF_PARENT_ADJ) { cA = Ia; cP = pa; cC = Ic; }
    else {
      const int slot = Map::ld(L.par_slot);
      if (slot >= 0) {
        acc_add27<RA>(lp(TM.l_acc + slot * TM.acc_words, RA(0)), SL, Ia, pa);
        rbi_acc<RC>(lp(TM.l_acc + slot * TM.acc_words + TM.acc_ic_word, RC(0)), SL, Ic);
      }
    }
  };
  if (team_contact) {   // zero the blocks that CRBA fills sparsely; padding dofs get an identity diagonal
    const int nkk = nbo * (nbo + 1) / 2 * 9;
    for (int k = 0; k < nkk; ++k) Mkk[k * SL] = RS(0);
    for (int k = n_od; k < 3 * nbo; ++k) Mkk[(btri(k / 3, k / 3) + (k % 3) * 4) * SL] = RS(1);
    for (int k = 0; k < nbo * nbt * 9; ++k) Ck[k * SL] = RS(0);
    if (role == 0) {
      const int nb9 = nbt * (nbt + 1) / 2 * 9;
      for (int k = 0; k < nb9; ++k) Bt[k * STM] = RS(0);
      for (int k = n_td; k < nt3; ++k) Bt[(btri(k / 3, k / 3) + (k % 3) * 4) * STM] = RS(1);
    }
  }
  // ---- pass 2a: subtrees ---------------------------------------------------------------------------------------------
  for (int k = n_loc - 1; k >= n_trunk; --k) pass2_link(k, (char*)own_rec(k, 0, RC(0)), (char*)own_rec(k, VOFF, RA(0)), SL);
  // attachment accumulators: sum of the four roles' partial accumulators
  if constexpr (Map::ROLE_WARPS) {   // role 0 (the only reader) sums them
    __syncthreads();
    if (role == 0) {
      for (int s = 0; s < TM.n_att; ++s) {
        RA* pa = lp(TM.l_acc + s * TM.acc_words, RA(0));
        const RA* p1 = (const RA*)Map::role_base(TM, tb, 1) + (size_t)(TM.l_acc + s * TM.acc_words) / RAW * SL + lane;
        const RA* p2 = (const RA*)Map::role_base(TM, tb, 2) + (size_t)(TM.l_acc + s * TM.acc_words) / RAW * SL + lane;
        const RA* p3 = (const RA*)Map::role_base(TM, tb, 3) + (size_t)(TM.l_acc + s * TM.acc_words) / RAW * SL + lane;
#pragma unroll 9
        for (int k = 0; k < 27; ++k) pa[k * SL] = (pa[k * SL] + p1[k * SL]) + (p2[k * SL] + p3[k * SL]);
        RC* pc = lp(TM.l_acc + s * TM.acc_words + TM.acc_ic_word, RC(0));
        const RC* c1 = (const RC*)Map::role_base(TM, tb, 1) + (size_t)(TM.l_acc + s * TM.acc_words + TM.acc_ic_word) / RCW * SL + lane;
        const RC* c2 = (const RC*)Map::role_base(TM, tb, 2) + (size_t)(TM.l_acc + s * TM.acc_words + TM.acc_ic_word) / RCW * SL + lane;
        const RC* c3 = (const RC*)Map::role_base(TM, tb, 3) + (size_t)(TM.l_acc + s * TM.acc_words + TM.acc_ic_word) / RCW * SL + lane;
#pragma unroll
        for (int k = 0; k < 10; ++k) pc[k * SL] = (pc[k * SL] + c1[k * SL]) + (c2[k * SL] + c3[k * SL]);
      }
    }
  } else {   // every lane of the team ends with the total
    for (int s = 0; s < TM.n_att; ++s) {
      RA* pa = lp(TM.l_acc + s * TM.acc_words, RA(0));
      for (int k = 0; k < 27; ++k) pa[k * SL] = team_sum(pa[k * SL], tmask);
      RC* pc = lp(TM.l_acc + s * TM.acc_words + TM.acc_ic_word, RC(0));
      for (int k = 0; k < 10; ++k) pc[k * SL] = team_sum(pc[k * SL], tmask);
    }
  }
  // ---- pass 2b + base + pass 3a: role 0 finishes the trunk -------------------------------------------------------------
  RA* const tabase = tvbase + 6 * STM;     // base acceleration (6 RA) published for the subtrees
  const RA dtA = RA(P.dt);
  auto pass3_link = [&](const int k, RA* const urec, RA* const vrec, const int ST, Sv<RA>& a_prev) {
    const TeamLink& L = mytl[k];
    const int fl = Map::ld(L.flags);
    const int lpar = Map::ld(L.lpar);
    Sv<RA> a;
    if (fl & TDS_TF_PARENT_ADJ) a = a_prev;
    else if (lpar < 0) a = ld6<RA>(tabase, STM);
    else if (lpar < n_trunk) a = ld6<RA>(tp(TM.t_link + lpar * LWD + VOFF, RA(0)), STM);
    else a = ld6<RA>(lp(TM.l_link + (lpar - n_trunk) * LWD + VOFF, RA(0)), SL);
    if (!(fl & TDS_LF_FIXED)) {
      const Sv<RA> c = ld6<RA>(vrec, ST);
      const Sv<RA> U = ld6<RA>(urec, ST);
      a = a + c;
      const RA qdd = urec[6 * ST] * (urec[7 * ST] - dot(U, a));
      const Sv<RA> S = cvt_sv<RA>(S_of(k));
      a.top = axpy(S.top, qdd, a.top);
      a.bot = axpy(S.bot, qdd, a.bot);
      const int qdi_ = Map::ld(L.qd_idx), ld_ = Map::ld(L.ldof);
      if (mode == MODE_FD) { if (live && io.qdd_out) io.qdd_out[(size_t)qdi_ * ns + e] = (float)qdd; }
      else { float& r = qd_ref(k, qdi_, ld_); r = (float)(RA(r) + qdd * dtA); }
    }
    st6<RA>(vrec, ST, a);
    a_prev = a;
  };
  if (role == 0) {
    for (int k = n_trunk - 1; k >= 0; --k) pass2_link(k, (char*)trunk_rec(k, 0, RC(0)), (char*)trunk_rec(k, VOFF, RA(0)), STM);
    // base acceleration (forward_dynamics.hpp:218-243)
    Sv<RA> a_prev;
    Sv<RC> base_acc_b; base_acc_b.top = v3<RC>(RC(0), RC(0), RC(0)); base_acc_b.bot = base_acc_b.top;
    if (M.floating) {
      Abi<RA> Ach; Sv<RA> pch; Rbi<RC> Icch;
      Ach.I = {RA(0), RA(0), RA(0), RA(0), RA(0), RA(0)}; Ach.M = Ach.I;
      Ach.H.xx = Ach.H.xy = Ach.H.xz = Ach.H.yx = Ach.H.yy = Ach.H.yz = Ach.H.zx = Ach.H.zy = Ach.H.zz = RA(0);
      pch.top = v3<RA>(RA(0), RA(0), RA(0)); pch.bot = pch.top;
      Icch.m = RC(0); Icch.h = v3<RC>(RC(0), RC(0), RC(0)); Icch.I = {RC(0), RC(0), RC(0), RC(0), RC(0), RC(0)};
      if (n_trunk > 0 && Map::ld(mytl[0].lpar) < 0 && (Map::ld(mytl[0].flags) & TDS_TF_PARENT_ADJ)) { abi_add(Ach, cA); pch = pch + cP; rbi_add(Icch, cC); }
      if (TM.base_slot >= 0) {
        Abi<RA> sa; Sv<RA> sp;
        acc_ld27<RA>(lp(TM.l_acc + TM.base_slot * TM.acc_words, RA(0)), SL, sa, sp);
        abi_add(Ach, sa); pch = pch + sp;
        rbi_add(Icch, ld_rbi<RC>(lp(TM.l_acc + TM.base_slot * TM.acc_words + TM.acc_ic_word, RC(0)), SL));
      }
      const M3<RA> Rt = cvt<RA>(transpose(Rb));
      Abi<RA> Ab;
      {
        Rbi<RA> rbb = model_rbi_of<RA>(M.base_rbi);
        Ab = abi_from_rbi(rbb);
        Abi<RA> Arot;
        Arot.I = rot_sym(Rt, Ach.I); Arot.M = rot_sym(Rt, Ach.M); Arot.H = rot_gen(Rt, Ach.H);
        abi_add(Ab, Arot);
      }
      Sv<RA> pb;
      {   // gyroscopic bias, kinematics.hpp:54-61
        const M3<RA> RbA = cvt<RA>(Rb);
        M3<RA> Ic0;
        Ic0.xx = RA(M.base_inertia_com[0]); Ic0.xy = RA(M.base_inertia_com[1]); Ic0.xz = RA(M.base_inertia_com[2]);
        Ic0.yx = RA(M.base_inertia_com[3]); Ic0.yy = RA(M.base_inertia_com[4]); Ic0.yz = RA(M.base_inertia_com[5]);
        Ic0.zx = RA(M.base_inertia_com[6]); Ic0.zy = RA(M.base_inertia_com[7]); Ic0.zz = RA(M.base_inertia_com[8]);
        const M3<RA> Iw = rot_gen(RbA, Ic0);
        const V3<RA> wb = v3<RA>(RA(tqd[0]), RA(tqd[STM]), RA(tqd[2 * STM]));
        pb.top = cross(wb, mul(Iw, wb)) + mul(Rt, pch.top);
        pb.bot = mul(Rt, pch.bot);
      }
      if (team_contact) {   // base block of M (mass_matrix.hpp:114-120) in the base frame
        Rbi<RC> Ib = model_rbi_of<RC>(M.base_rbi);
        const M3<RC> RtC = transpose(Rb);
        Rbi<RC> rot; rot.m = Icch.m; rot.h = mul(RtC, Icch.h); rot.I = rot_sym(RtC, Icch.I);
        rbi_add(Ib, rot);
        const RS z = RS(0);
        RS* b00 = Bt + btri(0, 0) * STM; RS* b10 = Bt + btri(1, 0) * STM; RS* b11 = Bt + btri(1, 1) * STM;
        b00[0] = RS(Ib.I.xx); b00[3 * STM] = RS(Ib.I.xy); b00[4 * STM] = RS(Ib.I.yy); b00[6 * STM] = RS(Ib.I.xz); b00[7 * STM] = RS(Ib.I.yz); b00[8 * STM] = RS(Ib.I.zz);
        b10[0] = z;                b10[STM] = RS(Ib.h.z);      b10[2 * STM] = RS(-Ib.h.y);
        b10[3 * STM] = RS(-Ib.h.z); b10[4 * STM] = z;           b10[5 * STM] = RS(Ib.h.x);
        b10[6 * STM] = RS(Ib.h.y);  b10[7 * STM] = RS(-Ib.h.x); b10[8 * STM] = z;
        b11[0] = RS(Ib.m); b11[3 * STM] = z; b11[4 * STM] = RS(Ib.m); b11[6 * STM] = z; b11[7 * STM] = z; b11[8 * STM] = RS(Ib.m);
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
        M3<RC> C = neg(H3);
        M3<RC> Dm = inv3(sub(M3m, mul(mul(C, Ainv), H3)));
        M3<RC> AinvBD = mul(mul(Ainv, H3), Dm);
        M3<RC> Ii = add(Ainv, mul(mul(AinvBD, C), Ainv));
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
    st6<RA>(tabase, STM, a_prev);
    for (int k = 0; k < n_trunk; ++k) pass3_link(k, trunk_rec(k, UOFF, RA(0)), trunk_rec(k, VOFF, RA(0)), STM, a_prev);
    if (M.floating) {   // forward_dynamics.hpp:317-322 (gravity added un-rotated), integrator.hpp:153-163
      const RC qb[6] = {base_acc_b.top.x, base_acc_b.top.y, base_acc_b.top.z, base_acc_b.bot.x + RC(P.gravity[0]),
                        base_acc_b.bot.y + RC(P.gravity[1]), base_acc_b.bot.z + RC(P.gravity[2])};
#pragma unroll
      for (int k = 0; k < 6; ++k) {
        if (mode == MODE_FD) { if (live && io.qdd_out) io.qdd_out[(size_t)k * ns + e] = (float)qb[k]; }
        else tqd[k * STM] = (float)(RC(tqd[k * STM]) + qb[k] * RC(P.dt));
      }
    }
  }
  Map::sync();
  TDST_PHASE();  // 3
  // ---- pass 3b: subtrees ---------------------------------------------------------------------------------------------------
  {
    Sv<RA> a_prev; a_prev.top = v3<RA>(RA(0), RA(0), RA(0)); a_prev.bot = a_prev.top;
    for (int k = n_trunk; k < n_loc; ++k) pass3_link(k, own_rec(k, UOFF, RA(0)), own_rec(k, VOFF, RA(0)), SL, a_prev);
  }
  if constexpr (!Map::ROLE_WARPS) __syncwarp();
  TDST_PHASE();  // 4
  if (mode == MODE_FD) return;

  // ---- contact solve: leaf-first block elimination ---------------------------------------------------------------------------
  RS* const dk = lp(TM.l_dinv, RS(0));
  RS* const dt_ = tp(TM.t_dinv, RS(0));
  RS* const wk = lp(TM.l_w, RS(0));
  RS* const wt = tp(TM.t_wt, RS(0));
  RS* const Pk = lp(TM.l_P, RS(0));
  const bool solve = (mode == MODE_FULL) && any_contact;   // uniform over the threads that meet at the barriers below
  auto factor_trunk = [&]() {   // trunk block: S = L_t L_t^T
    for (int bi = 0; bi < nbt; ++bi)
      for (int bj = 0; bj <= bi; ++bj) {
        B9<RS> Ab = ldb<RS>(Bt + btri(bi, bj) * STM, STM);
        for (int bk = 0; bk < bj; ++bk) gemm_nt_sub(Ab, ldb<RS>(Bt + btri(bi, bk) * STM, STM), ldb<RS>(Bt + btri(bj, bk) * STM, STM));
        if (bj < bi) stb<RS>(Bt + btri(bi, bj) * STM, STM, mul_linvT(Ab, ldl6<RS>(dt_ + bj * 6 * STM, STM)));
        else stl6<RS>(dt_ + bi * 6 * STM, STM, chol3_inv(Ab));
      }
    for (int k = 0; k < nt3; ++k) wt[k * STM] = RS(0);
  };
  if (solve && team_contact) {
    // own block: M_kk = L_k L_k^T (blocked), G = L_k^-1 C
    for (int bi = 0; bi < nbo; ++bi) {
      for (int bj = 0; bj <= bi; ++bj) {
        B9<RS> Ab = ldb<RS>(Mkk + btri(bi, bj) * SL, SL);
        for (int bk = 0; bk < bj; ++bk) gemm_nt_sub(Ab, ldb<RS>(Mkk + btri(bi, bk) * SL, SL), ldb<RS>(Mkk + btri(bj, bk) * SL, SL));
        if (bj < bi) stb<RS>(Mkk + btri(bi, bj) * SL, SL, mul_linvT(Ab, ldl6<RS>(dk + bj * 6 * SL, SL)));
        else stl6<RS>(dk + bi * 6 * SL, SL, chol3_inv(Ab));
      }
      for (int bt = 0; bt < nbt; ++bt) {
        B9<RS> a = ldb<RS>(Ck + (bi * nbt + bt) * 9 * SL, SL);
        for (int bk = 0; bk < bi; ++bk) gemm_nn_sub(a, ldb<RS>(Mkk + btri(bi, bk) * SL, SL), ldb<RS>(Ck + (bk * nbt + bt) * 9 * SL, SL));
        stb<RS>(Ck + (bi * nbt + bt) * 9 * SL, SL, linv_mul(ldl6<RS>(dk + bi * 6 * SL, SL), a));
      }
    }
    // partial Schur complement P = G^T G (lower blocks) of this role, summed over the roles
    for (int b1 = 0; b1 < nbt; ++b1)
      for (int b2 = 0; b2 <= b1; ++b2) {
        B9<RS> acc;
#pragma unroll
        for (int q = 0; q < 9; ++q) acc.a[q] = RS(0);
        for (int bo = 0; bo < nbo; ++bo) {
          const B9<RS> g1 = ldb<RS>(Ck + (bo * nbt + b1) * 9 * SL, SL), g2 = ldb<RS>(Ck + (bo * nbt + b2) * 9 * SL, SL);
#pragma unroll
          for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c) acc.a[r * 3 + c] += g1.a[r] * g2.a[c] + g1.a[3 + r] * g2.a[3 + c] + g1.a[6 + r] * g2.a[6 + c];
        }
        if constexpr (Map::ROLE_WARPS) stb<RS>(Pk + btri(b1, b2) * SL, SL, acc);   // summed by role 0 below
        else {
#pragma unroll
          for (int q = 0; q < 9; ++q) acc.a[q] = team_sum(acc.a[q], tmask);
          if (role == 0) {
            RS* pb = Bt + btri(b1, b2) * STM;
#pragma unroll
            for (int q = 0; q < 9; ++q) pb[q * STM] -= acc.a[q];
          }
        }
      }
    if constexpr (!Map::ROLE_WARPS) { if (role == 0) factor_trunk(); }
    for (int k = 0; k < 3 * nbo; ++k) wk[k * SL] = RS(0);
  }
  if constexpr (Map::ROLE_WARPS) {
    if (solve) __syncthreads();
    if (solve && team_contact && role == 0) {   // S = B - sum over the roles of G^T G, then factor it
      constexpr int RSW = (int)(sizeof(RS) / 4);
      const int nb9 = nbt * (nbt + 1) / 2 * 9;
      const RS* p1 = (const RS*)Map::role_base(TM, tb, 1) + (size_t)TM.l_P / RSW * SL + lane;
      const RS* p2 = (const RS*)Map::role_base(TM, tb, 2) + (size_t)TM.l_P / RSW * SL + lane;
      const RS* p3 = (const RS*)Map::role_base(TM, tb, 3) + (size_t)TM.l_P / RSW * SL + lane;
#pragma unroll 9
      for (int k = 0; k < nb9; ++k) Bt[k * STM] -= (Pk[k * SL] + p1[k * SL]) + (p2[k * SL] + p3[k * SL]);
      factor_trunk();
    }
    if (solve) __syncthreads();
  } else __syncwarp();
  TDST_PHASE();  // 5
  const int YW = TM.y_words / (int)(sizeof(RS) / 4);   // RS elements per candidate: own part (3 nbo_max*3) then trunk part
  const int no3max = 3 * TM.nbo_max;
  if (solve && team_contact) {
    const V3<RC> nbv = v3<RC>(-pn.x, -pn.y, -pn.z);                     // world_normal_on_b
    const V3<RC> f1 = v3<RC>(RC(M.fr1[0]), RC(M.fr1[1]), RC(M.fr1[2]));
    const V3<RC> f2 = v3<RC>(RC(M.fr2[0]), RC(M.fr2[1]), RC(M.fr2[2]));
    // Y rows of this role's active candidates
    const int npts = TM.n_pts[role];
    for (int lpt = 0; lpt < npts; ++lpt) {
      const RC* pc = lp(TM.l_con + lpt * 5 * RCW, RC(0));
      const int kl = (int)pc[4 * SL];
      if (kl < -1) continue;           // not penetrating
      RS* const Yo = lp(TM.l_Y, RS(0)) + (size_t)lpt * YW * SL;          // own dofs: [dof][rhs]
      RS* const Yt = Yo + no3max * 3 * SL;                                // trunk dofs
      const V3<RC> xc = ld3<RC>(pc, SL);
      const RC dist = pc[3 * SL];
      for (int k = 0; k < YW; ++k) Yo[k * SL] = RS(0);
      V3<RC> vel = v3<RC>(RC(0), RC(0), RC(0));
      if (M.floating) {   // jacobian.hpp:39-58 with r = x_c
        const V3<RC> cols[6] = {v3<RC>(RC(0), -xc.z, xc.y), v3<RC>(xc.z, RC(0), -xc.x), v3<RC>(-xc.y, xc.x, RC(0)),
                                v3<RC>(RC(1), RC(0), RC(0)), v3<RC>(RC(0), RC(1), RC(0)), v3<RC>(RC(0), RC(0), RC(1))};
#pragma unroll
        for (int k = 0; k < 6; ++k) {
          Yt[(3 * k) * SL] = RS(dot(nbv, cols[k])); Yt[(3 * k + 1) * SL] = RS(dot(f1, cols[k])); Yt[(3 * k + 2) * SL] = RS(dot(f2, cols[k]));
          vel = vel + cols[k] * RC(tqd[k * STM]);
        }
      }
      for (int j = kl; j >= 0; j = Map::ld(mytl[j].lpar)) {   // jacobian.hpp:63-80
        const int lj = Map::ld(mytl[j].ldof);
        if (lj < 0) continue;
        const Sv<RC> S = S_of(j);
        const V3<RC> col = S.bot + cross(S.top, xc);
        RS* dst = lj >= n_td ? Yo + (3 * (lj - n_td)) * SL : Yt + (3 * lj) * SL;
        dst[0] = RS(dot(nbv, col)); dst[SL] = RS(dot(f1, col)); dst[2 * SL] = RS(dot(f2, col));
        vel = vel + col * RC(qd_ref(j, Map::ld(mytl[j].qd_idx), lj));
      }
      RS* const cs = lp(TM.l_conS, RS(0)) + lpt * 12 * SL;   // b[3], x[3], y.y[3], 1/A_ii[3]   (mb_constraint_solver.hpp:299-345)
      cs[0] = RS((RC(1) + RC(P.restitution)) * dot(nbv, vel) - RC(P.erp) * dist / RC(P.dt));
      cs[SL] = RS(dot(f1, vel));
      cs[2 * SL] = RS(dot(f2, vel));
      cs[3 * SL] = RS(0); cs[4 * SL] = RS(0); cs[5 * SL] = RS(0);
      // y_own = L_k^-1 r_own
      for (int bi = 0; bi < nbo; ++bi) {
        B9<RS> a = ldb<RS>(Yo + bi * 9 * SL, SL);
        for (int bk = 0; bk < bi; ++bk) gemm_nn_sub(a, ldb<RS>(Mkk + btri(bi, bk) * SL, SL), ldb<RS>(Yo + bk * 9 * SL, SL));
        stb<RS>(Yo + bi * 9 * SL, SL, linv_mul(ldl6<RS>(dk + bi * 6 * SL, SL), a));
      }
      // y_t = L_t^-1 (r_t - G^T y_own)
      for (int bt = 0; bt < nbt; ++bt) {
        B9<RS> a = ldb<RS>(Yt + bt * 9 * SL, SL);
        for (int bo = 0; bo < nbo; ++bo) {   // a -= G[bo][bt]^T * y_own[bo]
          const B9<RS> g = ldb<RS>(Ck + (bo * nbt + bt) * 9 * SL, SL), y = ldb<RS>(Yo + bo * 9 * SL, SL);
#pragma unroll
          for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c) a.a[r * 3 + c] -= g.a[r] * y.a[c] + g.a[3 + r] * y.a[3 + c] + g.a[6 + r] * y.a[6 + c];
        }
        for (int bk = 0; bk < bt; ++bk) gemm_nn_sub(a, ldb<RS>(Bt + btri(bt, bk) * STM, STM), ldb<RS>(Yt + bk * 9 * SL, SL));
        stb<RS>(Yt + bt * 9 * SL, SL, linv_mul(ldl6<RS>(dt_ + bt * 6 * STM, STM), a));
      }
      // A_ii = y.y + cfm is constant during the sweep: keep y.y and 1 / A_ii per row
      for (int blk = 0; blk < 3; ++blk) {
        RS yy = RS(0);
        for (int k = 0; k < 3 * nbo; ++k) { const RS y = Yo[(3 * k + blk) * SL]; yy += y * y; }
        for (int k = 0; k < nt3; ++k) { const RS y = Yt[(3 * k + blk) * SL]; yy += y * y; }
        cs[(6 + blk) * SL] = yy;
        cs[(9 + blk) * SL] = RS(1) / (yy + RS(P.cfm));
      }
    }
  }
  if (solve) {
    TDST_PHASE();  // 6
    // projected Gauss-Seidel in the reference's row order (solve_pgs, mb_constraint_solver.hpp:101-142,417-436).
    // A row is relaxed by the role that owns its contact; the trunk part of w = Y p is shared through wt, which the
    // owner updates in place.
    const RS mu = RS(P.friction);
    auto relax_row = [&](const int g, const int blk) {
      const int lpt = TM.cand_lpt[g];
      RS* const cs = lp(TM.l_conS, RS(0)) + lpt * 12 * SL;
      const RS* yo = lp(TM.l_Y, RS(0)) + (size_t)lpt * YW * SL + blk * SL;     // element k at yo[3k * SL]
      const RS* yt = yo + no3max * 3 * SL;
      RS yw0 = RS(0), yw1 = RS(0), yw2 = RS(0);
      for (int b = 0; b < nbo; ++b) {
        yw0 += yo[(9 * b) * SL] * wk[(3 * b) * SL]; yw1 += yo[(9 * b + 3) * SL] * wk[(3 * b + 1) * SL]; yw2 += yo[(9 * b + 6) * SL] * wk[(3 * b + 2) * SL];
      }
      for (int b = 0; b < nbt; ++b) {
        yw0 += yt[(9 * b) * SL] * wt[(3 * b) * STM]; yw1 += yt[(9 * b + 3) * SL] * wt[(3 * b + 1) * STM]; yw2 += yt[(9 * b + 6) * SL] * wt[(3 * b + 2) * STM];
      }
      const RS yw = (yw0 + yw1) + yw2;
      const RS x_old = cs[(3 + blk) * SL];
      RS x = (cs[blk * SL] - yw + cs[(6 + blk) * SL] * x_old) * cs[(9 + blk) * SL];
      if (blk == 0) {
        x = x < RS(0) ? RS(0) : x;
        x = x > RS(100000) ? RS(100000) : x;
      } else {
        RS s = cs[3 * SL];
        s = s < RS(0) ? RS(0) : s;
        const RS lim = mu * s;
        x = x < -lim ? -lim : x;
        x = x > lim ? lim : x;
      }
      cs[(3 + blk) * SL] = x;
      const RS dx = x - x_old;
      for (int b = 0; b < nbo; ++b) {
        wk[(3 * b) * SL] += dx * yo[(9 * b) * SL];
        wk[(3 * b + 1) * SL] += dx * yo[(9 * b + 3) * SL];
        wk[(3 * b + 2) * SL] += dx * yo[(9 * b + 6) * SL];
      }
      for (int k = 0; k < nt3; ++k) wt[k * STM] += dx * yt[(3 * k) * SL];
    };
    int last_owner = -1;
    for (int it = 0; it < P.pgs_iterations; ++it) {
      for (int blk = 0; blk < 3; ++blk) {
        if constexpr (Map::ROLE_WARPS) {
          // every candidate in order: a CTA barrier separates consecutive rows of different owners (rows of one
          // owner follow in program order)
          for (int g = 0; g < TM.n_cand; ++g) {
            const int owner = TM.cand_owner[g];
            if (owner != last_owner && last_owner >= 0) __syncthreads();
            last_owner = owner;
            if (role == owner && ((team_active >> g) & 1ull)) relax_row(g, blk);
          }
        } else {   // the active candidates of this environment
          unsigned long long rem = team_active;
          while (rem) {
            const int g = __ffsll((long long)rem) - 1;
            rem &= rem - 1;
            if (role == TM.cand_owner[g]) relax_row(g, blk);
            __syncwarp(tmask);   // publish w_trunk before the next row reads it
          }
        }
      }
    }
    if constexpr (Map::ROLE_WARPS) __syncthreads();
    TDST_PHASE();  // 7
    // dqd = L^-T w (mb_constraint_solver.hpp:476-497): z_t = L_t^-T w_t by role 0, then z_k = L_k^-T (w_k - G z_t)
    if (role == 0 && team_contact) {
      for (int bi = nbt - 1; bi >= 0; --bi) {
        RS a0 = wt[(3 * bi) * STM], a1 = wt[(3 * bi + 1) * STM], a2 = wt[(3 * bi + 2) * STM];
        for (int bk = bi + 1; bk < nbt; ++bk) {
          const B9<RS> Lb = ldb<RS>(Bt + btri(bk, bi) * STM, STM);
          const RS z0 = wt[(3 * bk) * STM], z1 = wt[(3 * bk + 1) * STM], z2 = wt[(3 * bk + 2) * STM];
          a0 -= Lb.a[0] * z0 + Lb.a[3] * z1 + Lb.a[6] * z2;
          a1 -= Lb.a[1] * z0 + Lb.a[4] * z1 + Lb.a[7] * z2;
          a2 -= Lb.a[2] * z0 + Lb.a[5] * z1 + Lb.a[8] * z2;
        }
        const L6<RS> li = ldl6<RS>(dt_ + bi * 6 * STM, STM);
        wt[(3 * bi) * STM] = li.i00 * a0 + li.i10 * a1 + li.i20 * a2;
        wt[(3 * bi + 1) * STM] = li.i11 * a1 + li.i21 * a2;
        wt[(3 * bi + 2) * STM] = li.i22 * a2;
      }
    }
    if constexpr (Map::ROLE_WARPS) __syncthreads();
    else __syncwarp(tmask);
    if (team_contact) {
      for (int bo = 0; bo < nbo; ++bo) {   // w_k -= G z_t
        RS a0 = wk[(3 * bo) * SL], a1 = wk[(3 * bo + 1) * SL], a2 = wk[(3 * bo + 2) * SL];
        for (int bt = 0; bt < nbt; ++bt) {
          const B9<RS> g = ldb<RS>(Ck + (bo * nbt + bt) * 9 * SL, SL);
          const RS z0 = wt[(3 * bt) * STM], z1 = wt[(3 * bt + 1) * STM], z2 = wt[(3 * bt + 2) * STM];
          a0 -= g.a[0] * z0 + g.a[1] * z1 + g.a[2] * z2;
          a1 -= g.a[3] * z0 + g.a[4] * z1 + g.a[5] * z2;
          a2 -= g.a[6] * z0 + g.a[7] * z1 + g.a[8] * z2;
        }
        wk[(3 * bo) * SL] = a0; wk[(3 * bo + 1) * SL] = a1; wk[(3 * bo + 2) * SL] = a2;
      }
      for (int bi = nbo - 1; bi >= 0; --bi) {
        RS a0 = wk[(3 * bi) * SL], a1 = wk[(3 * bi + 1) * SL], a2 = wk[(3 * bi + 2) * SL];
        for (int bk = bi + 1; bk < nbo; ++bk) {
          const B9<RS> Lb = ldb<RS>(Mkk + btri(bk, bi) * SL, SL);
          const RS z0 = wk[(3 * bk) * SL], z1 = wk[(3 * bk + 1) * SL], z2 = wk[(3 * bk + 2) * SL];
          a0 -= Lb.a[0] * z0 + Lb.a[3] * z1 + Lb.a[6] * z2;
          a1 -= Lb.a[1] * z0 + Lb.a[4] * z1 + Lb.a[7] * z2;
          a2 -= Lb.a[2] * z0 + Lb.a[5] * z1 + Lb.a[8] * z2;
        }
        const L6<RS> li = ldl6<RS>(dk + bi * 6 * SL, SL);
        wk[(3 * bi) * SL] = li.i00 * a0 + li.i10 * a1 + li.i20 * a2;
        wk[(3 * bi + 1) * SL] = li.i11 * a1 + li.i21 * a2;
        wk[(3 * bi + 2) * SL] = li.i22 * a2;
      }
      // qd -= z : own dofs by their role, trunk dofs by role 0
      for (int k = n_trunk; k < n_loc; ++k) {
        const int lj = Map::ld(mytl[k].ldof);
        if (lj >= 0) { float& r = tqd[Map::ld(mytl[k].qd_idx) * STM]; r = (float)(RS(r) - wk[(lj - n_td) * SL]); }
      }
      if (role == 0) {
        if (M.floating) for (int k = 0; k < 6; ++k) tqd[k * STM] = (float)(RS(tqd[k * STM]) - wt[k * STM]);
        for (int k = 0; k < n_trunk; ++k) {
          const int lj = Map::ld(mytl[k].ldof);
          if (lj >= 0) { float& r = tqd[Map::ld(mytl[k].qd_idx) * STM]; r = (float)(RS(r) - wt[lj * STM]); }
        }
      }
    }
  }
  if constexpr (!Map::ROLE_WARPS) __syncwarp();
  TDST_PHASE();  // 8

  // ---- integrate_euler with qdd = 0 (integrator.hpp:10-133), reward / done, write back -----------------------------------------
  RC up_z = RC(1);
  if (role == 0 && M.floating) {
    const RC h = RC(0.5) * RC(P.dt);
    RC qx = RC(tq[0]), qy = RC(tq[STM]), qz = RC(tq[2 * STM]), qw = RC(tq[3 * STM]);
    const RC w0 = RC(tqd[0]), w1 = RC(tqd[STM]), w2 = RC(tqd[2 * STM]);
    const RC dw = (-qx * w0 - qy * w1 - qz * w2) * h;
    const RC dx = (qw * w0 + qz * w1 - qy * w2) * h;
    const RC dy = (qw * w1 + qx * w2 - qz * w0) * h;
    const RC dz = (qw * w2 + qy * w0 - qx * w1) * h;
    qx += dx; qy += dy; qz += dz; qw += dw;
    const RC len = sqrt_t(qx * qx + qy * qy + qz * qz + qw * qw);
    qx /= len; qy /= len; qz /= len; qw /= len;
    tq[0] = (float)qx; tq[STM] = (float)qy; tq[2 * STM] = (float)qz; tq[3 * STM] = (float)qw;
    for (int k = 0; k < 3; ++k) tq[(4 + k) * STM] = (float)(RC(tq[(4 + k) * STM]) + RC(tqd[(3 + k) * STM]) * RC(P.dt));
    up_z = RC(1) - RC(2) * (qx * qx + qy * qy) / (qx * qx + qy * qy + qz * qz + qw * qw);
  }
  for (int k = k_first; k < n_loc; ++k) {
    const TeamLink& L = mytl[k];
    if (Map::ld(L.flags) & TDS_LF_FIXED) continue;
    const int qi = Map::ld(L.q_idx), qdi = Map::ld(L.qd_idx), ld = Map::ld(L.ldof);
    float& qr = q_ref(k, qi, ld);
    qr = (float)(RC(qr) + RC(qd_ref(k, qdi, ld)) * RC(P.dt));
  }
  // reward / done read coordinates that another role may have just corrected and integrated (on a fixed base every
  // subtree hangs off the base, so q[0..6] need not be role 0's)
  if (E.reward_kind) Map::sync();
  int done_i = 0;
  if (role == 0) {
    bool done = false;
    if (E.reward_kind == 1) {   // laikago_environment2.h:130-171 (fixed-base emulation; q0..5 are trunk coordinates)
      const float x = tq[0], z = tq[2 * STM];
      const float upz = cosf(tq[3 * STM]) * cosf(tq[4 * STM]);
      done = (upz < 0.6f) || (z < 0.2f);
      if (io.reward && live) io.reward[e] = done ? 0.f : x;
    } else if (E.reward_kind == 2) {
      const float x = tq[4 * STM], z = tq[6 * STM];
      done = ((float)up_z < 0.6f) || (z < 0.2f);
      if (io.reward && live) io.reward[e] = done ? 0.f : x;
    } else if (E.reward_kind == 3) {   // ant_environment2.h:75-105: done = z < 0.26, reward = (x' - x)/dt, which integrate_euler makes the x velocity
      done = tq[2 * STM] < 0.26f;
      if (io.reward && live) io.reward[e] = done ? 0.f : tqd[0];
    }
    if (io.done && E.reward_kind && live) io.done[e] = done ? 1.f : 0.f;
    done_i = done ? 1 : 0;
  }
  // role 0's done flag to every role
  if constexpr (Map::ROLE_WARPS) {
    if (role == 0) amask[(2 * TT) * STM] = (unsigned)done_i;
    __syncthreads();
    done_i = (int)amask[(2 * TT) * STM];
  } else done_i = __shfl_sync(tmask, done_i, team * TT);
  const bool reset = done_i && E.auto_reset;
  if constexpr (!Map::ROLE_WARPS) __syncwarp();
  if (live) {
#pragma unroll 4
    for (int k = role; k < M.n_q; k += TT) io.q_out[(size_t)k * ns + e] = reset ? E.reset_q[k] : tq[k * STM];
#pragma unroll 4
    for (int k = role; k < M.n_qd; k += TT) io.qd_out[(size_t)k * ns + e] = reset ? 0.f : tqd[k * STM];
  }
  TDST_PHASE();  // 9
}
#undef TDST_PHASE

#ifndef TDS_TEAM_KERNEL_ONLY   // launchers: not part of the host-compiled kernel source (tests/cpp/team_host.cpp)
// Host side: one launch of tds_team_step_kernel<Map, RA, RC, RS, SM>.  The dynamic shared-memory limit is raised
// once per instance and device.
template <class Map, typename RA, typename RC, typename RS, bool SM>
cudaError_t launch_team_step(const TeamModel* TM, const TeamLink* tl, const DevModel* M, const SimParams* P,
                             const EnvParams* E, const StepIO* io, int mode, int use_pd, char* gscratch, size_t smem,
                             cudaStream_t stream) {
  auto k = tds_team_step_kernel<Map, RA, RC, RS, SM>;
  cudaError_t err = cudaSuccess;
  static size_t smem_set_dev[64] = {0}; int dev_ = 0; cudaGetDevice(&dev_); size_t& smem_set = smem_set_dev[dev_ & 63];
  if (smem > 48 * 1024 && smem > smem_set) {
    err = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (Map::MAX_CARVEOUT && err == cudaSuccess)
      err = cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    if (err == cudaSuccess) smem_set = smem;
  }
  if (err != cudaSuccess) return err;
  const int tiles = (io->n + Map::STM - 1) / Map::STM;
  k<<<tiles, Map::THREADS, smem, stream>>>(*TM, tl, *M, *P, *E, *io, mode, use_pd, gscratch);
  return cudaGetLastError();
}

// precision 0: RA fp32 / RC fp64 / RS fp32, 1: all fp64, 2: all fp32 (tds_stepw.cu)
template <class Map>
int launch_team_step(const TeamModel* TM, const TeamLink* tl, const DevModel* M, const SimParams* P, const EnvParams* E,
                     const StepIO* io, int mode, int use_pd, int precision, char* gscratch, int use_smem,
                     cudaStream_t stream) {
  const size_t smem = use_smem ? Map::tile_bytes(*TM) : 0;
#define TDST_LAUNCH(RA, RC, RS)                                                                                      \
  (use_smem ? launch_team_step<Map, RA, RC, RS, true>(TM, tl, M, P, E, io, mode, use_pd, gscratch, smem, stream)    \
            : launch_team_step<Map, RA, RC, RS, false>(TM, tl, M, P, E, io, mode, use_pd, gscratch, smem, stream))
  const cudaError_t err = precision == 0 ? TDST_LAUNCH(float, double, float)
                        : precision == 1 ? TDST_LAUNCH(double, double, double)
                                         : TDST_LAUNCH(float, float, float);
#undef TDST_LAUNCH
  return (int)err;
}
#endif  // TDS_TEAM_KERNEL_ONLY

}  // namespace tdsteam
