// Team ("sub-warp") decomposition of one environment over T lanes: the kinematic tree is cut into a TRUNK
// (ancestor-closed set of links at the root, processed by lane 0 of the team) and SUBTREES hanging off the
// trunk, distributed over the T lanes.  Host side: partition + per-role link tables + scratch layout.
// Device side: tds_team_step.cuh (step body), run by tds_stept.cu (lane teams) and tds_stepr.cu (role warps).
#pragma once
#include <string.h>

#include <algorithm>
#include <vector>

#include "tds_model.h"
#include "tds_types.h"

#define TDS_TEAM_T 4
#define TDS_TEAM_MAXK 28   // local links per role (trunk + own)
#define TDS_TEAM_MAXC 48   // candidate contact points per model

// local link flags (in addition to TDS_LF_FIXED/REVOLUTE/PRISMATIC/XT_IDENT)
#define TDS_TF_PARENT_ADJ 64     // parent is the previous link in this role's processing order (register carry)
#define TDS_TF_CHILD_ADJ 128     // the next link in processing order is a child that carries into this link
#define TDS_TF_PARENT_TRUNK 256  // own link whose parent is a trunk link (or the base): contribution goes to an attachment slot

struct TeamLink {            // one record per (role, local position); read with __ldg
  double XT[12];
  double axis[3];
  double rbic[10];           // mass, com (link frame), inertia about the com (xx,xy,xz,yy,yz,zz)
  float stiffness, damping;
  int link;                  // global link index
  int lpar;                  // local position of the parent (-1: base)
  int flags;
  int jtype;
  int q_idx, qd_idx;         // global coordinates (for HBM I/O)
  int ldof;                  // local dof index: trunk dofs [0, n_td), own dofs [n_td, ...); -1 for fixed joints
  int acc_slot;              // accumulator receiving this link's non-carried children (-1: none)
  int par_slot;              // accumulator this link adds its contribution to (-1: carry or dropped)
  int xw_slot;               // slot where (R, p) is kept for non-adjacent children (-1: none); trunk: team region
  int g_begin, g_end;        // global geom range
  int cand_begin;            // global candidate index of this link's first contact point
  int lpt_begin;             // role-local candidate index of this link's first contact point
  int act_idx;               // action index driving this joint (-1: none)
  int pad;
};

struct TeamModel {
  int T;
  int n_trunk, n_td, nbt;            // trunk links, trunk dofs (6 base dofs first when floating), trunk dof blocks
  int n_loc[TDS_TEAM_T];             // local links per role (trunk + own)
  int n_od[TDS_TEAM_T], nbo[TDS_TEAM_T];
  int n_pts[TDS_TEAM_T];             // candidate contact points per role (role 0: trunk + own)
  int base_pts;                      // candidate points on base geoms (role 0)
  int kmax, n_od_max, nbo_max, n_pts_max;
  int n_att;                         // attachment accumulators (trunk nodes / base receiving subtrees): slots [0, n_att)
  int n_acc;                         // accumulator slots per lane (attachment + internal)
  int base_slot;                     // accumulator slot of the floating base (-1)
  int n_xw_team, n_xw_lane;
  int n_cand;
  int cand_owner[TDS_TEAM_MAXC];
  int cand_lpt[TDS_TEAM_MAXC];
  // layout, 4-byte words.  team region: [word][team] ; lane region: [word][lane]
  int t_q, t_qd, t_tau, t_S, t_link, t_xw, t_O, t_B, t_dinv, t_wt, t_total;
  int l_q, l_qd, l_tau, l_S, l_link, l_xw, l_acc, l_M, l_C, l_dinv, l_w, l_con, l_conS, l_Y, l_P, l_total;
  int link_words, acc_words, acc_ic_word, y_words;
  int n_q, n_qd, floating, has_plane, n_links;
};

// Partition + tables.  Returns 0 on success; >0 if the model has no useful decomposition (use the one-lane kernel);
// <0 on capacity errors.
static inline int tds_build_team(const DevModel* D, const EnvParams* E, TeamModel* TM, std::vector<TeamLink>* table) {
  memset(TM, 0, sizeof(*TM));
  const int T = TDS_TEAM_T, n = D->n_links;
  TM->T = T;
  TM->n_q = D->n_q; TM->n_qd = D->n_qd; TM->floating = D->floating; TM->has_plane = D->has_plane; TM->n_links = n;
  std::vector<std::vector<int>> children(n + 1);  // children[0] = children of the base (-1)
  for (int i = 0; i < n; ++i) children[D->parent[i] + 1].push_back(i);
  std::vector<int> size(n, 1);
  for (int i = n - 1; i >= 0; --i) if (D->parent[i] >= 0) size[D->parent[i]] += size[i];
  std::vector<char> trunk(n, 0);
  std::vector<int> roots = children[0];
  // grow the trunk until there are at least T subtrees (split the largest subtree while that helps)
  while ((int)roots.size() < T) {
    int best = -1;
    for (int r = 0; r < (int)roots.size(); ++r)
      if (!children[roots[r] + 1].empty() && (best < 0 || size[roots[r]] > size[roots[best]])) best = r;
    if (best < 0) break;
    int rl = roots[best];
    trunk[rl] = 1;
    roots.erase(roots.begin() + best);
    for (int c : children[rl + 1]) roots.push_back(c);
  }
  if ((int)roots.size() < 2) return 1;  // a chain: nothing to distribute
  // chains leading to a single big subtree are better in the trunk than replicated nowhere: keep as is.
  std::sort(roots.begin(), roots.end(), [&](int a, int b) { return size[a] != size[b] ? size[a] > size[b] : a < b; });
  std::vector<int> owner(n, -1), load(T, 0);
  for (int r : roots) {
    int lane = (int)(std::min_element(load.begin(), load.end()) - load.begin());
    load[lane] += size[r];
    std::vector<int> stack{r};
    while (!stack.empty()) {
      int x = stack.back(); stack.pop_back();
      owner[x] = lane;
      for (int c : children[x + 1]) stack.push_back(c);
    }
  }
  int n_trunk = 0;
  for (int i = 0; i < n; ++i) if (trunk[i]) ++n_trunk;
  TM->n_trunk = n_trunk;
  // local lists: trunk (ascending) then own (ascending)
  std::vector<std::vector<int>> list(T);
  for (int r = 0; r < T; ++r) {
    for (int i = 0; i < n; ++i) if (trunk[i]) list[r].push_back(i);
    for (int i = 0; i < n; ++i) if (!trunk[i] && owner[i] == r) list[r].push_back(i);
    if ((int)list[r].size() > TDS_TEAM_MAXK) return -1;
    TM->n_loc[r] = (int)list[r].size();
    TM->kmax = std::max(TM->kmax, TM->n_loc[r]);
  }
  // dofs
  int n_td = D->floating ? 6 : 0;
  std::vector<int> ldof(n, -1);
  for (int i = 0; i < n; ++i) if (trunk[i] && !(D->flags[i] & TDS_LF_FIXED)) ldof[i] = n_td++;
  TM->n_td = n_td; TM->nbt = (n_td + 2) / 3;
  for (int r = 0; r < T; ++r) {
    int k = n_td;
    for (int i : list[r]) if (!trunk[i] && !(D->flags[i] & TDS_LF_FIXED)) ldof[i] = k++;
    TM->n_od[r] = k - n_td; TM->nbo[r] = (TM->n_od[r] + 2) / 3;
    TM->n_od_max = std::max(TM->n_od_max, TM->n_od[r]);
    TM->nbo_max = std::max(TM->nbo_max, TM->nbo[r]);
  }
  // attachment accumulators: trunk links / base that have non-trunk children, plus trunk links with non-adjacent trunk children
  std::vector<int> att_slot(n + 1, -1);   // index link+1
  int n_acc = 0;
  for (int i = 0; i < n; ++i) {
    if (trunk[i]) continue;
    int p = D->parent[i];
    if (p >= 0 && !trunk[p]) continue;
    if (p < 0 && !D->floating) continue;     // fixed base: contribution is dropped
    if (att_slot[p + 1] < 0) att_slot[p + 1] = n_acc++;
  }
  TM->n_att = n_acc;
  // candidate contact points (global enumeration order: base geoms, then links in order)
  std::vector<int> cand_begin(n + 1, 0), npts(n + 1, 0);
  {
    int c = 0;
    for (int li = -1; li < n; ++li) {
      cand_begin[li + 1] = c;
      for (int g = D->geom_begin[li + 1]; g < D->geom_begin[li + 2]; ++g) {
        int k = D->g_type[g] == TDSG_SPHERE ? 1 : (D->g_type[g] == TDSG_CAPSULE ? 2 : 0);
        c += k; npts[li + 1] += k;
      }
    }
    if (!D->has_plane) c = 0;
    if (c > TDS_TEAM_MAXC) return -2;
    TM->n_cand = c;
  }
  TM->base_pts = D->has_plane ? npts[0] : 0;
  // per-role tables
  table->assign((size_t)T * TDS_TEAM_MAXK, TeamLink());
  std::vector<int> internal_slots(T, 0), xw_lane(T, 0);
  int xw_team = 0;
  std::vector<int> trunk_xw(n, -1);
  int trunk_internal = 0;
  std::vector<int> trunk_acc(n + 1, -1);
  for (int r = 0; r < T; ++r) {
    std::vector<int> lpos(n, -1);
    for (int k = 0; k < TM->n_loc[r]; ++k) lpos[list[r][k]] = k;
    int lpt = (r == 0) ? TM->base_pts : 0;
    std::vector<int> own_acc(n, -1), own_xw(n, -1);
    for (int k = 0; k < TM->n_loc[r]; ++k) {
      const int i = list[r][k];
      TeamLink& L = (*table)[(size_t)r * TDS_TEAM_MAXK + k];
      memset(&L, 0, sizeof(L));
      memcpy(L.XT, D->XT[i], sizeof(L.XT));
      memcpy(L.axis, D->axis[i], sizeof(L.axis));
      memcpy(L.rbic, D->rbic[i], sizeof(L.rbic));
      L.stiffness = D->stiffness[i]; L.damping = D->damping[i];
      L.link = i;
      const int p = D->parent[i];
      L.lpar = p >= 0 ? lpos[p] : -1;
      L.jtype = D->jtype[i];
      L.q_idx = D->q_idx[i]; L.qd_idx = D->qd_idx[i];
      L.ldof = ldof[i];
      L.flags = D->flags[i] & (TDS_LF_FIXED | TDS_LF_REVOLUTE | TDS_LF_PRISMATIC | TDS_LF_XT_IDENT);
      L.acc_slot = -1; L.par_slot = -1; L.xw_slot = -1; L.act_idx = -1;
      L.g_begin = D->geom_begin[i + 1]; L.g_end = D->geom_begin[i + 2];
      L.cand_begin = cand_begin[i + 1];
      const bool mine = trunk[i] ? (r == 0) : true;
      L.lpt_begin = lpt;
      if (mine && D->has_plane) lpt += npts[i + 1];
      if (E) for (int a = 0; a < E->n_act; ++a) if (E->act_link[a] == i) L.act_idx = a;
      const bool parent_trunk_or_base = (p < 0) || trunk[p];
      if (!trunk[i] && parent_trunk_or_base) {
        L.flags |= TDS_TF_PARENT_TRUNK;
        L.par_slot = att_slot[p + 1];          // -1 for a fixed base: dropped
      } else if (L.lpar == k - 1 && !(k == n_trunk && !trunk[i])) {
        L.flags |= TDS_TF_PARENT_ADJ;          // carry (for k == 0 the parent is the base)
      }
      if (k == 0 && p < 0 && trunk[i]) L.flags |= TDS_TF_PARENT_ADJ;
    }
    // second pass: accumulator / xw slots for non-adjacent children inside this role's list
    for (int k = 0; k < TM->n_loc[r]; ++k) {
      const int i = list[r][k];
      TeamLink& L = (*table)[(size_t)r * TDS_TEAM_MAXK + k];
      if (L.flags & (TDS_TF_PARENT_ADJ | TDS_TF_PARENT_TRUNK)) continue;
      const int p = D->parent[i];
      if (p < 0) {           // a trunk root after the first (the trunk grew into several children of the base)
        if (!D->floating) continue;          // fixed base: dropped, as for subtrees
        if (trunk_acc[0] < 0) trunk_acc[0] = (att_slot[0] >= 0) ? att_slot[0] : (TM->n_att + 64 + trunk_internal++);
        L.par_slot = trunk_acc[0];           // the base reads it through base_slot
        continue;
      }
      // parent p is in this list, non adjacent
      if (trunk[i]) {        // trunk-internal branch (role independent numbering)
        if (trunk_acc[p + 1] < 0) trunk_acc[p + 1] = (att_slot[p + 1] >= 0) ? att_slot[p + 1] : (TM->n_att + 64 + trunk_internal++);
        L.par_slot = trunk_acc[p + 1];
      } else {
        if (own_acc[p] < 0) own_acc[p] = TM->n_att + internal_slots[r]++;
        L.par_slot = own_acc[p];
      }
    }
    (void)own_xw;
  }
  // renumber: attachment [0, n_att) | own-internal (max over roles) | trunk-internal
  int own_int_max = 0;
  for (int r = 0; r < T; ++r) own_int_max = std::max(own_int_max, internal_slots[r]);
  for (auto& L : *table) if (L.par_slot >= TM->n_att + 64) L.par_slot = L.par_slot - 64 + own_int_max;
  TM->n_acc = TM->n_att + own_int_max + trunk_internal;
  TM->base_slot = D->floating ? att_slot[0] : -1;
  if (D->floating && TM->base_slot < 0 && trunk_acc[0] >= 0) TM->base_slot = trunk_acc[0] - 64 + own_int_max;
  // receiving side: acc_slot of a link = the par_slot its non-carried children use
  for (int r = 0; r < T; ++r)
    for (int k = 0; k < TM->n_loc[r]; ++k) {
      TeamLink& L = (*table)[(size_t)r * TDS_TEAM_MAXK + k];
      if (L.par_slot >= 0 && L.lpar >= 0) {
        TeamLink& Pp = (*table)[(size_t)r * TDS_TEAM_MAXK + L.lpar];
        Pp.acc_slot = L.par_slot;
      }
    }
  // every role's copy of a trunk link must agree on acc_slot (attachment totals arrive by butterfly in every lane)
  for (int k = 0; k < n_trunk; ++k) {
    int s = -1;
    for (int r = 0; r < T; ++r) s = std::max(s, (*table)[(size_t)r * TDS_TEAM_MAXK + k].acc_slot);
    for (int r = 0; r < T; ++r) (*table)[(size_t)r * TDS_TEAM_MAXK + k].acc_slot = s;
  }
  // CHILD_ADJ + xw slots
  for (int r = 0; r < T; ++r) {
    int xl = 0;
    for (int k = 0; k < TM->n_loc[r]; ++k) {
      TeamLink& L = (*table)[(size_t)r * TDS_TEAM_MAXK + k];
      if ((L.flags & TDS_TF_PARENT_ADJ) && L.lpar >= 0) (*table)[(size_t)r * TDS_TEAM_MAXK + L.lpar].flags |= TDS_TF_CHILD_ADJ;
    }
    for (int k = 0; k < TM->n_loc[r]; ++k) {
      TeamLink& L = (*table)[(size_t)r * TDS_TEAM_MAXK + k];
      if (L.flags & TDS_TF_PARENT_ADJ) continue;
      if (L.lpar < 0) continue;              // base: kept in the team region anyway
      TeamLink& Pp = (*table)[(size_t)r * TDS_TEAM_MAXK + L.lpar];
      const int pi = Pp.link;
      if (trunk[pi]) { if (trunk_xw[pi] < 0) trunk_xw[pi] = xw_team++; }
      else if (Pp.xw_slot < 0) Pp.xw_slot = xl++;
    }
    xw_lane[r] = xl;
  }
  for (int r = 0; r < T; ++r)
    for (int k = 0; k < n_trunk; ++k) (*table)[(size_t)r * TDS_TEAM_MAXK + k].xw_slot = trunk_xw[list[r][k]];
  TM->n_xw_team = xw_team;
  for (int r = 0; r < T; ++r) TM->n_xw_lane = std::max(TM->n_xw_lane, xw_lane[r]);
  // candidate points -> owner role / role-local index
  for (int r = 0; r < T; ++r) {
    int lp = (r == 0) ? TM->base_pts : 0;
    for (int k = 0; k < TM->n_loc[r]; ++k) {
      const TeamLink& L = (*table)[(size_t)r * TDS_TEAM_MAXK + k];
      const bool mine = (k < n_trunk) ? (r == 0) : true;
      if (!mine || !D->has_plane) continue;
      for (int c = 0; c < npts[L.link + 1]; ++c) {
        TM->cand_owner[L.cand_begin + c] = r;
        TM->cand_lpt[L.cand_begin + c] = lp++;
      }
    }
    TM->n_pts[r] = lp;
    TM->n_pts_max = std::max(TM->n_pts_max, lp);
  }
  for (int c = 0; c < TM->base_pts; ++c) { TM->cand_owner[c] = 0; TM->cand_lpt[c] = c; }
  return 0;
}

// Scratch layout: team region [word][team] (one column per environment of the warp) and lane region [word][lane].
static inline void tds_build_team_layout(TeamModel* TM, int size_ra, int size_rc, int size_rs) {
  const int ra = size_ra / 4, rc = size_rc / 4, rs = size_rs / 4;
  auto even = [](int x) { return (x + 1) & ~1; };
  // link record: rigid inertia about O (10 RC) | U (6), 1/D, u (8 RA) | v / c / a (6 RA); every word range is
  // accessed through ONE element size (the 4- and 8-byte views interleave lanes differently)
  TM->link_words = even(10 * rc + 14 * ra);
  TM->acc_ic_word = even(27 * ra);
  TM->acc_words = even(TM->acc_ic_word + 10 * rc);
  const int nt3 = 3 * TM->nbt, no3 = 3 * TM->nbo_max;
  int w = 0;
  // ---- team region ----
  TM->t_q = w; w += TM->n_q;                 // trunk coordinates live at their global index (simple, small)
  TM->t_qd = w; w += TM->n_qd;
  TM->t_tau = w; w += TM->n_qd;
  w = even(w);
  TM->t_O = w; w += 16 * rc;                 // O[3], plane_off, Rb[9], pad
  TM->t_S = w; w += TM->n_trunk * 6 * rc;
  w = even(w);
  TM->t_link = w; w += TM->n_trunk * TM->link_words;
  w = even(w);
  TM->t_xw = w; w += (TM->n_xw_team + 1) * 12 * rc + 12 * ra;   // slot 0: base; then base velocity + acceleration (RA)
  w = even(w);
  TM->t_B = w; w += (TM->nbt * (TM->nbt + 1) / 2) * 9 * rs;
  w = even(w);
  TM->t_dinv = w; w += TM->nbt * 6 * rs;
  w = even(w);
  TM->t_wt = w; w += nt3 * rs;
  w = even(w);
  TM->t_total = w;
  // ---- lane region ----
  w = 0;
  const int kown = TM->kmax - TM->n_trunk;
  TM->l_q = TM->l_qd = TM->l_tau = 0;        // (coordinates live in the team region)
  TM->l_S = w; w += kown * 6 * rc;
  w = even(w);
  TM->l_xw = w; w += TM->n_xw_lane * 12 * rc;
  w = even(w);
  {   // accumulators; the role-warp kernel reuses the region for its partial Schur complement (l_P)
    const int acc_region = (TM->n_acc > 0 ? TM->n_acc : 1) * TM->acc_words;
    const int p_region = (TM->nbt * (TM->nbt + 1) / 2) * 9 * rs;
    TM->l_acc = w; TM->l_P = w; w += acc_region > p_region ? acc_region : p_region;
  }
  w = even(w);
  TM->l_M = w; w += (TM->nbo_max * (TM->nbo_max + 1) / 2) * 9 * rs;
  w = even(w);
  TM->l_C = w; w += TM->nbo_max * TM->nbt * 9 * rs;       // C, later G = L^-1 C
  w = even(w);
  TM->l_dinv = w; w += (TM->nbo_max > 0 ? TM->nbo_max : 1) * 6 * rs;
  w = even(w);
  TM->l_w = w; w += no3 * rs + 2;
  w = even(w);
  const int npt = TM->n_pts_max > 0 ? TM->n_pts_max : 1;
  TM->l_con = w; w += npt * 5 * rc;
  w = even(w);
  TM->l_conS = w; w += npt * 12 * rs;
  w = even(w);
  TM->y_words = (no3 + nt3) * 3 * rs;
  const int link_region = kown * TM->link_words;
  const int y_region = npt * TM->y_words;
  TM->l_link = w; TM->l_Y = w;
  w += link_region > y_region ? link_region : y_region;
  w = even(w);
  TM->l_total = w;
}
