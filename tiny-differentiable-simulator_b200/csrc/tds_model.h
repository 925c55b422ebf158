// Host-side "model compiler" back end: flat model (include/tds_b200_model.h) -> DevModel
// (constant-bank kernel parameter) + per-environment scratch layout.
#pragma once
#include <math.h>
#include <string.h>

#include "tds_b200_model.h"
#include "tds_types.h"

#ifndef __CUDACC__
#define TDS_HOST_INLINE static inline
#else
#define TDS_HOST_INLINE static inline __host__
#endif

// MultiBodyConstraintSolver::plane_space, src/mb_constraint_solver.hpp:506-520 (evaluated once on the
// host: the contact normal of every plane contact is the constant -plane_normal).
TDS_HOST_INLINE void tds_plane_space(const double* n, double* p, double* q) {
  double n_sqr = n[2] * n[2];
  int mz = n_sqr > 0.5;
  double a = n[1] * n[1] + (mz ? n_sqr : n[0] * n[0]);
  double k = sqrt(a);
  p[0] = mz ? 0.0 : -n[1] * k;
  p[1] = mz ? -n[2] * k : n[0] * k;
  p[2] = mz ? n[1] * k : n[1] * k;
  q[0] = mz ? a * k : -n[2] * p[1];
  q[1] = mz ? -n[0] * p[2] : n[2] * p[0];
  q[2] = mz ? n[0] * p[1] : a * k;
}

// rigid-body inertia (mass, com, inertia about com) -> (m, h = m com, I about the link origin),
// i.e. the blocks of ArticulatedBodyInertia(rbi), src/math/inertia.hpp:114-119.
TDS_HOST_INLINE void tds_rbi_pack(const double* rec /* mass, com[3], inertia[9] */, double* out) {
  double m = rec[0];
  const double* c = rec + 1;
  const double* I = rec + 4;
  // H = cross(com); I_o = inertia + H H^T m ; H H^T = (c.c) 1 - c c^T
  double cc = c[0] * c[0] + c[1] * c[1] + c[2] * c[2];
  out[0] = m;
  out[1] = (m * c[0]); out[2] = (m * c[1]); out[3] = (m * c[2]);
  out[4] = (I[0] + m * (cc - c[0] * c[0]));
  out[5] = (0.5 * (I[1] + I[3]) - m * c[0] * c[1]);
  out[6] = (0.5 * (I[2] + I[6]) - m * c[0] * c[2]);
  out[7] = (I[4] + m * (cc - c[1] * c[1]));
  out[8] = (0.5 * (I[5] + I[7]) - m * c[1] * c[2]);
  out[9] = (I[8] + m * (cc - c[2] * c[2]));
}

// (mass, com, inertia about com) kept as given, symmetric part of the inertia.
TDS_HOST_INLINE void tds_rbic_pack(const double* rec, double* out) {
  out[0] = rec[0];
  out[1] = rec[1]; out[2] = rec[2]; out[3] = rec[3];
  const double* I = rec + 4;
  out[4] = I[0]; out[5] = 0.5 * (I[1] + I[3]); out[6] = 0.5 * (I[2] + I[6]);
  out[7] = I[4]; out[8] = 0.5 * (I[5] + I[7]); out[9] = I[8];
}

// Returns 0 on success, <0 on unsupported / oversized models.
TDS_HOST_INLINE int tds_build_dev_model(const double* m, int n_doubles, DevModel* D) {
  if (n_doubles < TDSM_HEADER || (int)m[TDSM_H_MAGIC] != TDSM_MAGIC) return -1;
  memset(D, 0, sizeof(*D));
  D->n_links = (int)m[TDSM_H_NLINKS];
  D->floating = (int)m[TDSM_H_FLOATING];
  D->n_q = (int)m[TDSM_H_NQ];
  D->n_qd = (int)m[TDSM_H_NQD];
  D->n_geoms = (int)m[TDSM_H_NGEOMS];
  D->n_vis = (int)m[TDSM_H_NVIS];
  D->has_plane = (int)m[TDSM_H_HASPLANE];
  if (D->n_links < 0 || D->n_geoms < 0 || D->n_vis < 0 || D->n_q < 0 || D->n_qd < 0) return -1;
  if (D->n_links > TDS_MAX_LINKS || D->n_geoms > TDS_MAX_GEOMS) return -2;
  const double* base = m + TDSM_HEADER;
  const double* links = base + TDSM_BASE;
  const double* geoms = links + (size_t)D->n_links * TDSM_LINK;
  if (n_doubles < TDSM_HEADER + TDSM_BASE + D->n_links * TDSM_LINK + D->n_geoms * TDSM_GEOM + D->n_vis * TDSM_VIS) return -1;
  tds_rbi_pack(base, D->base_rbi);
  tds_rbic_pack(base, D->base_rbic);
  for (int k = 0; k < 9; ++k) D->base_inertia_com[k] = (float)base[4 + k];
  int n_acc = 0;
  for (int i = 0; i < D->n_links; ++i) D->acc_slot[i] = -1;
  D->base_acc = -1;
  for (int i = 0; i < D->n_links; ++i) {
    const double* l = links + (size_t)i * TDSM_LINK;
    int jt = (int)l[TDSM_L_JTYPE];
    if (jt < TDSJ_FIXED || jt > TDSJ_SPHERICAL) return -3;
    D->parent[i] = (int)l[TDSM_L_PARENT];
    if (D->parent[i] >= i) return -4;
    D->jtype[i] = jt;
    D->q_idx[i] = (int)l[TDSM_L_QIDX];
    D->qd_idx[i] = (int)l[TDSM_L_QDIDX];
    if (jt != TDSJ_FIXED && (D->q_idx[i] < 0 || D->q_idx[i] >= D->n_q || D->qd_idx[i] < 0 || D->qd_idx[i] >= D->n_qd)) return -1;
    if (jt == TDSJ_SPHERICAL && (D->q_idx[i] + 3 >= D->n_q || D->qd_idx[i] + 2 >= D->n_qd)) return -1;
    int fl = 0;
    D->s3_slot[i] = -1;
    if (jt == TDSJ_FIXED) fl |= TDS_LF_FIXED;
    else if (jt <= TDSJ_PRISMATIC_AXIS) fl |= TDS_LF_PRISMATIC;
    else if (jt == TDSJ_SPHERICAL) { fl |= TDS_LF_SPHERICAL; D->s3_slot[i] = D->n_sph++; D->world_only = 1; }
    else fl |= TDS_LF_REVOLUTE;
    if (D->parent[i] == i - 1) fl |= TDS_LF_PARENT_ADJ;
    D->flags[i] = fl;
    for (int k = 0; k < 3; ++k) D->axis[i][k] = l[TDSM_L_AXIS + k];
    for (int k = 0; k < 9; ++k) D->XT[i][k] = l[TDSM_L_XT_R + k];
    for (int k = 0; k < 3; ++k) D->XT[i][9 + k] = l[TDSM_L_XT_T + k];
    tds_rbi_pack(l + TDSM_L_MASS, D->rbi[i]);
    tds_rbic_pack(l + TDSM_L_MASS, D->rbic[i]);
    {
      const double* r = l + TDSM_L_XT_R;
      if (r[0] == 1.0 && r[4] == 1.0 && r[8] == 1.0 && r[1] == 0.0 && r[2] == 0.0 && r[3] == 0.0 && r[5] == 0.0 &&
          r[6] == 0.0 && r[7] == 0.0)
        D->flags[i] |= TDS_LF_XT_IDENT;
    }
    D->stiffness[i] = (float)l[TDSM_L_STIFFNESS];
    D->damping[i] = (float)l[TDSM_L_DAMPING];
  }
  for (int i = 0; i < D->n_links; ++i) {
    int p = D->parent[i];
    if (D->flags[i] & TDS_LF_PARENT_ADJ) {
      if (p >= 0) D->flags[p] |= TDS_LF_CHILD_ADJ;
    } else if (p >= 0) {
      if (D->acc_slot[p] < 0) D->acc_slot[p] = n_acc++;
    } else if (D->floating) {
      if (D->base_acc < 0) D->base_acc = n_acc++;
    }
  }
  D->n_acc = n_acc;
  // world transforms that must outlive the register carry: parents of non-adjacent children
  D->n_xw = 0;
  for (int i = 0; i < D->n_links; ++i) D->xw_slot[i] = -1;
  for (int i = 0; i < D->n_links; ++i) {
    int p = D->parent[i];
    if (!(D->flags[i] & TDS_LF_PARENT_ADJ) && p >= 0 && D->xw_slot[p] < 0) D->xw_slot[p] = D->n_xw++;
  }
  // common-frame origin: floating base -> base position; else the position of the first link that is not
  // reached through prismatic / fixed joints only (the root chain prefix)
  D->n_prefix = -1;
  if (!D->floating) {
    int k = 0;
    while (k < D->n_links && D->parent[k] == k - 1 && (D->flags[k] & (TDS_LF_PRISMATIC | TDS_LF_FIXED))) ++k;
    D->n_prefix = k;   // links 0..k-1 are translation-only; origin = world position of link k (or of link k-1's frame end)
  }
  int n_points = 0;
  for (int g = 0; g < D->n_geoms; ++g) {
    const double* gg = geoms + (size_t)g * TDSM_GEOM;
    D->g_link[g] = (int)gg[TDSM_G_LINK];
    D->g_type[g] = (int)gg[TDSM_G_TYPE];
    D->g_radius[g] = gg[TDSM_G_P];
    for (int k = 0; k < 3; ++k) D->g_t[g][k] = gg[TDSM_G_T + k];
    double hl = 0.5 * gg[TDSM_G_P + 1];
    for (int k = 0; k < 3; ++k) D->g_half[g][k] = gg[TDSM_G_R + k * 3 + 2] * hl;  // R_local * (0,0,L/2)
    if (D->g_type[g] == TDSG_SPHERE) n_points += 1;
    if (D->g_type[g] == TDSG_CAPSULE) n_points += 2;
    if (D->g_type[g] == TDSG_BOX) {
      // contact_plane_box, src/contact_point.hpp:164-198: a sphere of radius max(1e-2, Box::radius = 0) at each of the 8
      // corner points (+-dx, +-dy, +-dz), d = extent / 2 - radius (Box::get_corner_points, src/geometry.hpp:244-260)
      n_points += 8;
      const double r = 1e-2;
      for (int a = 0; a < 3; ++a) {
        const double d = 0.5 * gg[TDSM_G_P + a] - r;
        for (int k = 0; k < 3; ++k) D->g_box[g][a * 3 + k] = gg[TDSM_G_R + k * 3 + a] * d;   // column a of R_local, scaled
      }
      D->g_radius[g] = r;
      if (D->has_plane) D->world_only = 1;
    }
    // the contact stage implements plane x {sphere, capsule, box}.  The reference has no mesh COLLISION shapes at all
    // (TINY_MESH_TYPE is "only for visual shapes", src/geometry.hpp:34; its URDF loader drops them, urdf_to_multi_body.hpp:234-277,
    // and so does ours): a flat model carrying one is malformed rather than something to simulate - refuse it
    // (a PLANE shape on a link of the robot is legal: it has no contact function against the ground plane, only against the
    // spheres / capsules / boxes of ANOTHER multibody; its unit normal travels in g_half)
    if (D->g_type[g] == TDSG_PLANE) { for (int k = 0; k < 3; ++k) D->g_half[g][k] = gg[TDSM_G_P + k]; }
    else if (D->has_plane && D->g_type[g] != TDSG_SPHERE && D->g_type[g] != TDSG_CAPSULE && D->g_type[g] != TDSG_BOX) return -6;
  }
  if (D->has_plane && n_points > TDS_MAX_POINTS) return -2;
  D->max_contacts = D->has_plane ? n_points : 0;
  {  // geoms are enumerated base first, then link 0, 1, ...: ranges per link
    int g = 0;
    for (int li = -1; li < D->n_links; ++li) {
      D->geom_begin[li + 1] = g;
      while (g < D->n_geoms && D->g_link[g] == li) ++g;
    }
    D->geom_begin[D->n_links + 1] = g;
    if (g != D->n_geoms) return -5;  // geoms not grouped by link
  }
  {  // several multibodies in one world: candidate points between geoms of different multibodies, in the enumeration order of
     // World::compute_contacts_multi_body_internal (src/world.hpp:212-281): pairs (a < b), links of a, geoms, links of b, geoms
    const int want = (int)m[TDSM_H_NBODIES];
    D->n_bodies = 1;
    for (int i = 0; i < D->n_links; ++i) D->body_of[i] = 0;
    for (int g = 0; g < D->n_geoms; ++g) D->g_wslot[g] = -1;
    if (want > 1) {
      if (D->floating) return -7;
      int nbod = 0;
      for (int i = 0; i < D->n_links; ++i) {
        if (D->parent[i] < 0) D->body_of[i] = nbod++;
        else D->body_of[i] = D->body_of[D->parent[i]];
        if (i > 0 && D->body_of[i] < D->body_of[i - 1]) return -7;   // multibodies must be contiguous
      }
      if (nbod != want) return -7;
      D->n_bodies = nbod;
      int np = 0, ng = 0;
      for (int a = 0; a < nbod; ++a)
        for (int b = a + 1; b < nbod; ++b) {
          const int before = np;
          for (int ga = 0; ga < D->n_geoms; ++ga) {
            if (D->g_link[ga] < 0 || D->body_of[D->g_link[ga]] != a) continue;
            for (int gb = 0; gb < D->n_geoms; ++gb) {
              if (D->g_link[gb] < 0 || D->body_of[D->g_link[gb]] != b) continue;
              const int ta = D->g_type[ga], tb = D->g_type[gb];
              // CollisionDispatcher, src/contact_point.hpp:468-501: sphere x sphere, capsule x sphere, and sphere x capsule through
              // the swapped call; every other pair of shapes has no contact function
              int kinds[8], nk = 0;
              if (ta == TDSG_SPHERE && tb == TDSG_SPHERE) { kinds[0] = 0; nk = 1; }
              else if (ta == TDSG_CAPSULE && tb == TDSG_SPHERE) { kinds[0] = 1; kinds[1] = -1; nk = 2; }
              else if (ta == TDSG_SPHERE && tb == TDSG_CAPSULE) { kinds[0] = 2; kinds[1] = -2; nk = 2; }
              // a PLANE shape on a link (contact_plane_sphere / _capsule / _box, contact_point.hpp:97-198; the pose of the plane's
              // link is not used): 100 + point on the other shape; 200 + point when the plane is on b (the dispatcher's swapped call)
              else if (ta == TDSG_PLANE || tb == TDSG_PLANE) {
                const int other = ta == TDSG_PLANE ? tb : ta, base = ta == TDSG_PLANE ? 100 : 200;
                const int n_o = other == TDSG_SPHERE ? 1 : (other == TDSG_CAPSULE ? 2 : (other == TDSG_BOX ? 8 : 0));
                for (int k = 0; k < n_o; ++k) kinds[nk++] = base + k;
              }
              for (int k = 0; k < nk; ++k) {
                if (np >= TDS_MAX_PAIR_POINTS) return -2;
                D->pp_ga[np] = ga; D->pp_gb[np] = gb; D->pp_kind[np] = kinds[k]; ++np;
                if (D->g_wslot[ga] < 0) D->g_wslot[ga] = D->n_gw++;
                if (D->g_wslot[gb] < 0) D->g_wslot[gb] = D->n_gw++;
              }
            }
          }
          if (np > before) {
            if (ng >= TDS_MAX_PAIR_GROUPS) return -2;
            D->pg_begin[ng++] = before;
            if (np - before > D->max_pair_rows) D->max_pair_rows = np - before;
          }
        }
      D->pg_begin[ng] = np;
      D->n_pair_points = np; D->n_pair_groups = ng;
      D->world_only = 1;   // a forest of multibodies: the tree decompositions of the other kernels assume one root chain
    }
  }
  for (int k = 0; k < 3; ++k) D->plane_n[k] = m[TDSM_H_PLANE_N + k];
  D->plane_c = m[TDSM_H_PLANE_C];
  double nb[3] = {-D->plane_n[0], -D->plane_n[1], -D->plane_n[2]};
  tds_plane_space(nb, D->fr1, D->fr2);
  return 0;
}

// Number of candidate contact points (static per model: every sphere / capsule end emits one,
// src/contact_point.hpp:112-124,149-158).
TDS_HOST_INLINE int tds_num_contact_points(const DevModel* D) { return D->max_contacts; }

// Per-environment scratch layout in 4-byte words.  size_ra / size_rc = sizeof of the ABA / contact
// scalar.  The Y rows of the contact solve alias the per-link ABA region (dead after pass 3).
TDS_HOST_INLINE void tds_build_layout(DevModel* D, int size_ra, int size_rc, int size_rs, int max_contacts) {
  const int ra = size_ra / 4, rc = size_rc / 4, rs = size_rs / 4;
  const int n = D->n_qd;
  if (max_contacts >= 0 && max_contacts < D->max_contacts) D->max_contacts = max_contacts;
  int w = 0;
  auto even = [](int x) { return (x + 1) & ~1; };
  D->w_q = w; w += D->n_q;
  D->w_qd = w; w += n;
  D->w_tau = w; w += n;
  w = even(w);
  D->acc_ic_word = even(27 * ra);
  D->acc_words = even(D->acc_ic_word + 10 * rs);
  D->w_acc = w; w += D->n_acc * D->acc_words;
  w = even(w);
  D->w_xw = w; w += (D->n_links + 1) * 12 * rc;
  D->w_con = w; w += D->max_contacts * 5 * rc;
  w = even(w);
  D->w_M = w; w += (n * (n + 1) / 2) * rs;
  w = even(w);
  D->w_invd = w; w += n * rs;
  w = even(w);
  D->w_w = w; w += n * rs;
  w = even(w);
  D->w_conS = w; w += D->max_contacts * 6 * rs;
  w = even(w);
  D->link_words = 26 * ra;
  const int link_region = D->n_links * D->link_words;
  const int y_region = 3 * D->max_contacts * n * rs;
  D->w_link = w;
  D->w_Y = w;
  w += link_region > y_region ? link_region : y_region;
  w = even(w);
  D->w_total = w;
}

// Scratch layout of the world-frame kernel (tds_stepw.cu).
TDS_HOST_INLINE void tds_build_layout_w(DevModel* D, int size_ra, int size_rc, int size_rs, int max_contacts, int size_rq = 4) {
  const int ra = size_ra / 4, rc = size_rc / 4, rs = size_rs / 4, rq = size_rq / 4;   // rq: words of a state scalar (q, qd, tau)
  const int n = D->n_qd;
  if (max_contacts >= 0 && max_contacts < D->max_contacts) D->max_contacts = max_contacts;
  D->nb = (n + 2) / 3;
  const int n3 = 3 * D->nb;
  int w = 0;
  auto even = [](int x) { return (x + 1) & ~1; };
  D->x_q = w; w += D->n_q * rq;
  D->x_qd = w; w += n * rq;
  D->x_tau = w; w += n * rq;
  w = even(w);
  D->x_S = w; w += D->n_links * 6 * rc;                     // motion subspace in the common frame
  w = even(w);
  D->x_S3 = w; w += D->n_sph * 18 * rc;                     // the three columns of every spherical joint
  w = even(w);
  D->x_xw = w; w += (D->n_xw + 1) * 12 * rc;                // slot 0: base
  w = even(w);
  D->x_acc_ic_word = even(27 * ra);
  D->x_acc_words = even(D->x_acc_ic_word + 10 * rc);
  D->x_acc = w; w += D->n_acc * D->x_acc_words;
  w = even(w);
  D->x_con = w; w += D->max_contacts * 5 * rc;
  w = even(w);
  D->x_gw = w; w += D->n_gw * 12 * rc;                      // world centre + capsule half axis / the three box half axes, for the pair stage
  D->x_pcon = w; w += D->n_pair_points * 9 * rc;            // pair contacts: point on a [3], normal on b [3], distance, link a, link b
  w = even(w);
  D->x_M = w; w += (D->nb * (D->nb + 1) / 2) * 9 * rs;
  w = even(w);
  D->x_dinv = w; w += D->nb * 6 * rs;
  w = even(w);
  D->x_w = w; w += n3 * rs;
  w = even(w);
  const int rows = D->max_contacts > D->max_pair_rows ? D->max_contacts : D->max_pair_rows;   // rows of the largest LCP
  D->x_conS = w; w += rows * 6 * rs;
  w = even(w);
  // per-link: rigid inertia about the origin (10 RC), later reused for U (6 RA), invD, u ; v / c / a (6 RA)
  const int urec = (D->n_sph ? 30 : 8) * ra;                // spherical: U (18), D^-1 (9), u (3)
  const int first = 10 * rc > urec ? 10 * rc : urec;
  D->x_link_words = even(first + 6 * ra);
  const int link_region = D->n_links * D->x_link_words;
  const int y_region = rows * n3 * 3 * rs;
  D->x_link = w;
  D->x_Y = w;
  w += link_region > y_region ? link_region : y_region;
  w = even(w);
  D->x_total = w;
}

// Layout of the world-frame kernel's external-wrench instances (tds_stepw.cu, template flag EXT; DESIGN.md section 7.18): the layout D
// (built by tds_build_layout_w) followed by the links' wrench sums, 6 RA words per link, 16-byte aligned so that every scalar type
// addresses them.  Returns the region's first word and sets *x_total to the words per lane of the grown layout; D itself is unchanged.
TDS_HOST_INLINE int tds_ext_layout_w(const DevModel* D, int size_ra, int* x_total) {
  const int x_ext = (D->x_total + 3) & ~3;
  *x_total = x_ext + ((D->n_links * 6 * (size_ra / 4) + 3) & ~3);
  return x_ext;
}

// Layout of the world-frame kernel's dynamics-derivative instances (tds_stepw.cu, template flag DER; DESIGN.md section 7.23): the layout D
// followed by a_i and f_i of every link, 12 RC words per link, 16-byte aligned.  Returns the words per lane of the grown layout, whose last
// 12 RC n_links words the kernel addresses; D itself is unchanged.
TDS_HOST_INLINE int tds_der_layout_w(const DevModel* D, int size_rc) {
  return ((D->x_total + 3) & ~3) + D->n_links * 12 * (size_rc / 4);
}

// ---- physical parameter ids (include/tds_b200.h, tds_b200_set_physical_params_*) ----------------------------------------------------
// 0 friction, 1 restitution, 2 + 10 b + c body b (0 = base, i + 1 = link i; c: mass, com x y z, I_com xx xy xz yy yz zz),
// 2 + 10 (n_links + 1) + 2 i + c link i (c: joint stiffness, joint damping)
TDS_HOST_INLINE int tds_param_count(const DevModel* D) { return 2 + 10 * (D->n_links + 1) + 2 * D->n_links; }

// ids[0..k) -> slot map.  Returns 0, or -1 with *err set: an id out of range, an id given twice, a base id on a fixed-base model.
TDS_HOST_INLINE int tds_build_par_map(const DevModel* D, int k, const int* ids, ParMap* pm, const char** err) {
  memset(pm, 0, sizeof(*pm));
  pm->friction = pm->restitution = -1;
  for (int b = 0; b <= TDS_MAX_LINKS; ++b) for (int c = 0; c < 10; ++c) pm->body[b][c] = -1;
  for (int i = 0; i < TDS_MAX_LINKS; ++i) pm->joint[i][0] = pm->joint[i][1] = -1;
  const int n_ids = tds_param_count(D), j0 = 2 + 10 * (D->n_links + 1);
  if (k < 0 || (k > 0 && !ids)) { *err = "bad parameter count"; return -1; }
  pm->n = k;
  for (int s = 0; s < k; ++s) {
    const int id = ids[s];
    if (id < 0 || id >= n_ids) { *err = "parameter id out of range"; return -1; }
    short* slot = nullptr;
    int* islot = nullptr;
    if (id == 0) islot = &pm->friction;
    else if (id == 1) islot = &pm->restitution;
    else if (id < j0) {
      const int b = (id - 2) / 10;
      if (b == 0 && !D->floating) { *err = "base parameter on a fixed-base model (its base does not move)"; return -1; }
      slot = &pm->body[b][(id - 2) % 10];
      if (b == 0) pm->any_base = 1;
    } else slot = &pm->joint[(id - j0) / 2][(id - j0) % 2];
    if ((islot && *islot >= 0) || (slot && *slot >= 0)) { *err = "parameter id given twice"; return -1; }
    if (islot) *islot = s; else *slot = (short)s;
  }
  return 0;
}
