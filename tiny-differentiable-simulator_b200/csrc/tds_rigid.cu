// The RigidBody path of the reference's World (SURVEY 8f.3): maximal-coordinate rigid bodies with ONE collision shape each,
// sequential-impulse contact solver.  One lane per world; a batch of worlds steps in one launch.
//   World::step                                   src/world.hpp:293-363 (the rigid-body half: :302-318, :336-340, :361-363)
//   RigidBody::apply_gravity / apply_force_impulse / apply_impulse / integrate   src/rigid_body.hpp:84-118
//   World::compute_contacts_rigid_body_internal   src/world.hpp:166-195 (pairs i < j through the dispatcher)
//   CollisionDispatcher                           src/contact_point.hpp:445-506 (direct or swapped call)
//   contact_sphere_sphere / plane_sphere / plane_capsule / plane_box / capsule_sphere   src/contact_point.hpp:44-438
//   RigidBodyConstraintSolver::resolve_collision  src/rb_constraint_solver.hpp:66-163 (the non-CppAD branch)
// State per body, fp64 in HBM as [13 * n_bodies][n_stride]: position [3], orientation xyzw [4], linear velocity [3],
// angular velocity [3].  Everything of a world lives in the lane's registers / local memory: the path is latency-bound
// scalar work (50 Gauss-Seidel sweeps over a handful of contacts), its HBM traffic is 2 x 104 B per body and step call.
#include <cuda_runtime.h>
#include <math.h>
#include <string.h>

#include "tds_math.cuh"
#include "tds_dual.cuh"
#include "tds_tape.cuh"
#include "tds_b200_model.h"

#define TDS_RIGID_MAX_BODIES 16
#define TDS_RIGID_MAX_CONTACTS 48

struct RigidWorld {                       // constant for all worlds of a batch (kernel parameter)
  int n_bodies;
  int type[TDS_RIGID_MAX_BODIES];         // TDSG_SPHERE / TDSG_PLANE / TDSG_CAPSULE / TDSG_BOX
  double mass[TDS_RIGID_MAX_BODIES];
  double p[TDS_RIGID_MAX_BODIES][4];      // sphere: radius; capsule: radius, length; box: extents [3]; plane: normal [3], constant
  double dt, gravity[3], friction, restitution, erp;
  int num_solver_iterations;
};

// Installed physical parameters (tds_b200_rigid_set_physical_params_*, DESIGN.md section 7.11): the slot of each quantity in the
// lane's value vector, or -1 = the RigidWorld's value.  Passed only to the PAR instances of the kernel.
struct RigidParMap {
  const double* values;                   // [k][n_stride] fp64, offset to the launch's first world
  const double* t_par;                    // JV instance: slot s of tangent j at t_par[(s * m + j) * n_stride + e], or null (zero tangent)
  double* grad;                           // taping instance: cotangents [k][n_stride] (offset like values), or null
  int n;                                  // installed parameters k (0: none)
  int friction, restitution;              // RigidWorld::friction / restitution
  int body[TDS_RIGID_MAX_BODIES][4];      // body b: c = 0 mass, c = 1..3 shape size p[b][c - 1]
};

// desc [n_bodies][6] = mass, shape (TDSG_*), p0..p3 -> RigidWorld (host).  The plane normal is normalised like Plane's constructor
// does (src/geometry.hpp:163-168).  Returns 0, -1 on an unknown shape, -2 when the contact list could overflow.
static inline int tds_rigid_world_from_desc(const double* desc, int n_bodies, RigidWorld* W) {
  memset(W, 0, sizeof(*W));
  W->n_bodies = n_bodies;
  for (int i = 0; i < n_bodies; ++i) {
    const double* d = desc + i * 6;
    const int t = (int)d[1];
    if (t != TDSG_SPHERE && t != TDSG_PLANE && t != TDSG_CAPSULE && t != TDSG_BOX) return -1;
    W->mass[i] = d[0]; W->type[i] = t;
    for (int k = 0; k < 4; ++k) W->p[i][k] = d[2 + k];
    if (t == TDSG_PLANE) {
      const double l = sqrt(d[2] * d[2] + d[3] * d[3] + d[4] * d[4]);
      for (int k = 0; k < 3; ++k) W->p[i][k] = d[2 + k] / l;
    }
  }
  // worst case of the contact list (every pair at the point count of its contact function): the kernel's list is fixed-size
  int worst = 0;
  for (int i = 0; i < n_bodies; ++i)
    for (int j = i + 1; j < n_bodies; ++j) {
      auto pts = [](int a, int b) { return (a == TDSG_SPHERE && b == TDSG_SPHERE) ? 1 : (a == TDSG_PLANE && b == TDSG_SPHERE) ? 1 : (a == TDSG_PLANE && b == TDSG_CAPSULE) ? 2
                                    : (a == TDSG_PLANE && b == TDSG_BOX) ? 8 : (a == TDSG_CAPSULE && b == TDSG_SPHERE) ? 2 : 0; };
      const int t = W->type[i], u = W->type[j];
      worst += pts(t, u) ? pts(t, u) : pts(u, t);
    }
  if (worst > TDS_RIGID_MAX_CONTACTS) return -2;
  // World defaults (world.hpp:65-72), RigidBodyConstraintSolver::erp_ (rb_constraint_solver.hpp:45)
  W->dt = 1.0 / 60.0; W->gravity[2] = -9.81; W->friction = 0.5; W->restitution = 0.0; W->erp = 0.1; W->num_solver_iterations = 1;
  return 0;
}

// parameter ids (include/tds_b200.h) -> RigidParMap (host; pointers left null).  nullptr, or the reason an id is refused.
static inline const char* tds_rigid_par_map(const RigidWorld& W, int k, const int* ids, RigidParMap* pm) {
  memset(pm, 0, sizeof(*pm));
  memset(pm->body, -1, sizeof(pm->body));
  pm->friction = pm->restitution = -1;
  pm->n = k;
  for (int s = 0; s < k; ++s) {
    const int id = ids[s];
    if (id < 0 || id >= 2 + 4 * W.n_bodies) return "id out of range";
    int* slot;
    if (id < 2) {
      slot = id == 0 ? &pm->friction : &pm->restitution;
    } else {
      const int b = (id - 2) / 4, c = (id - 2) % 4, t = W.type[b];
      if (t == TDSG_PLANE) return "a plane has no parameters";
      if (c == 0 && W.mass[b] == 0.0) return "the mass of a static body (model mass 0) is not a parameter";
      if (c > (t == TDSG_SPHERE ? 1 : t == TDSG_CAPSULE ? 2 : 3)) return "a size component the body's shape does not have";
      slot = &pm->body[b][c];
    }
    if (*slot >= 0) return "id given twice";
    *slot = s;
  }
  return nullptr;
}

// a value the host entry accepts for parameter id: finite; a mass or size > 0, friction and restitution >= 0
static inline bool tds_rigid_par_value_ok(int id, double v) {
  return isfinite(v) && (id >= 2 ? v > 0.0 : v >= 0.0);
}

namespace tdsrb {
using namespace tds;

// buffers of the taping instance (vector-Jacobian product of ONE step): cotangent g_out [13 nb][ns] -> g_state [13 nb][ns] and
// g_force [3 nb][ns] (may be null; g_state must not alias g_out: a chunk that overflowed is rerun from the same g_out).  tape / adj: cap nodes /
// adjoints per lane, interleaved by lane within a warp.  cap 0 or g_out null: values only (s_out), nothing recorded.
struct RigidVjpIO {
  const double* g_out; double* g_state; double* g_force;
  TapeNode* tape; double* adj; int cap; int* overflow;
};

// buffers of the Jacobian-vector product instance (JV, dual numbers; one lane per (world, tangent j = blockIdx.y + jac_dir0), the
// whole rollout): state entry r of tangent j is t_state[(r * m + j) * ns + e], force entry r t_force[(r * m + j) * ns + e] (either may
// be null: zero tangent); t_out [13 nb * m][ns] receives d state_out along tangent j at row r, column j
struct RigidJvpIO { const double* t_state; const double* t_force; double* t_out; int m; };
template <bool JV> struct RigidArg { typedef RigidVjpIO type; };
template <> struct RigidArg<true> { typedef RigidJvpIO type; };
// kernel argument of the instances without installed parameters: nothing
struct RigidNoPar {};
template <bool PAR> struct RigidParArg { typedef RigidNoPar type; };
template <> struct RigidParArg<true> { typedef RigidParMap type; };
// the lane's physical quantities in the PAR instances: installed values (seeded) or the RigidWorld's
template <typename T, bool PAR> struct RigidLanePar {};
template <typename T> struct RigidLanePar<T, true> { T mass[TDS_RIGID_MAX_BODIES], size[TDS_RIGID_MAX_BODIES][3], friction, restitution; };

template <typename T> struct Contact { V3<T> n, ra, rb; T dist; int a, b; };   // normal on b, point - position of a / b

// contact_sphere_sphere (contact_point.hpp:44-94) between two spheres given by centre and radius; pa / pb: the bodies' positions
template <typename T>
TDS_D void sphere_sphere(const V3<T>& ca, T ra, const V3<T>& cb, T rb, Contact<T>* cs, int& nc, int a, int b, const V3<T>& pa,
                         const V3<T>& pb, bool swap) {
  const V3<T> diff = ca - cb;
  const T len = sqrt_t(dot(diff, diff));
  if (!(len > T(1e-5)) || nc >= TDS_RIGID_MAX_CONTACTS) return;   // CONTACT_EPSILON
  const T dist = len - (ra + rb);
  const V3<T> n = diff * (T(1) / len);
  const V3<T> point_a = ca - n * ra;
  const V3<T> point_b = point_a - n * dist;
  Contact<T>& c = cs[nc++];
  c.dist = dist;
  if (!swap) { c.n = n; c.ra = point_a - pa; c.rb = point_b - pb; c.a = a; c.b = b; }
  else { c.n = v3<T>(-n.x, -n.y, -n.z); c.ra = point_b - pb; c.rb = point_a - pa; c.a = b; c.b = a; }   // dispatcher :478-492
}

// contact_plane_sphere (contact_point.hpp:97-124): plane = body a (its pose is not used), sphere centre c
template <typename T>
TDS_D void plane_sphere(const V3<T>& pn, T pc, const V3<T>& c, T r, Contact<T>* cs, int& nc, int a, int b, const V3<T>& pa,
                        const V3<T>& pb, bool swap) {
  if (nc >= TDS_RIGID_MAX_CONTACTS) return;
  const V3<T> mn = v3<T>(-pn.x, -pn.y, -pn.z);
  const T t = -(dot(c, mn) + pc);
  const V3<T> point_a = c + mn * t;
  const V3<T> point_b = c - pn * r;
  Contact<T>& k = cs[nc++];
  k.dist = t - r;
  if (!swap) { k.n = mn; k.ra = point_a - pa; k.rb = point_b - pb; k.a = a; k.b = b; }
  else { k.n = pn; k.ra = point_b - pb; k.rb = point_a - pa; k.a = b; k.b = a; }
}

// PAR: per-world physical parameters (DESIGN.md section 7.11).  Slot s of the lane is pm.values[s * ns + e], loaded once at the start
// into the lane's RigidLanePar (the model's value for every quantity without a slot), and every read site of a mass, a shape size,
// the friction or the restitution uses it.  The dual instance seeds slot s as direction 16 nb + s and writes it to column s of jac
// ([rows][k][ns]); the JV instance seeds it from pm.t_par; the taping instance makes it leaf 16 nb + s (after the state | force
// inputs, so g_state and g_force keep their layout) and writes its cotangent to pm.grad.  Seeded once per lane: a lane running
// `steps` steps gives the derivative of the whole rollout.  A body's static status (model mass 0) is structural, not a parameter.
template <typename T, typename TS, bool JV = false, bool PAR = false>
__global__ void __launch_bounds__(128) tds_rigid_step_kernel(const __grid_constant__ RigidWorld W, const TS* s_in,
                                                             TS* s_out, const TS* __restrict__ force, int steps,
                                                             int n, int ns, double* __restrict__ jac, int jac_dir0,
                                                             const typename RigidArg<JV>::type vio = {},
                                                             const __grid_constant__ typename RigidParArg<PAR>::type pm = {}) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  constexpr bool AD = is_dual<T>::value;
  constexpr bool TP = is_tape<T>::value;                     // taping instance: one lane per world, one step
  const int dir = AD ? (int)blockIdx.y + jac_dir0 : -1;      // differentiable instance: input direction of this lane
  const int nb = W.n_bodies;
  auto seed = [&](T x, int idx) -> T {   // d input_idx / d direction, or leaf idx of the tape, or the tangent's entry idx
    if constexpr (JV) return idx < 13 * nb ? jv_seed(x, vio.t_state, idx, vio.m, dir, ns, e) : jv_seed(x, vio.t_force, idx - 13 * nb, vio.m, dir, ns, e);
    else return ad_seed(x, idx, dir);
  };
  // (the instances without parameters keep their original statements: their code must not change)
  if constexpr (TP && PAR) tape_begin(vio.tape + ((size_t)(e >> 5) * vio.cap * 32 + (e & 31)), vio.g_out ? vio.cap : 0, vio.overflow, 16 * nb + pm.n);
  else if constexpr (TP) tape_begin(vio.tape + ((size_t)(e >> 5) * vio.cap * 32 + (e & 31)), vio.g_out ? vio.cap : 0, vio.overflow, 16 * nb);
  RigidLanePar<T, PAR> lp;
  if constexpr (PAR) {
    auto ld_par = [&](int slot, double model_v) -> T {   // one read per slot and lane, coalesced over the warp
      if (slot < 0) return T(model_v);
      const T x = T(pm.values[(size_t)slot * ns + e]);
      if constexpr (JV) return jv_seed(x, pm.t_par, slot, vio.m, dir, ns, e);
      else return ad_seed(x, 16 * nb + slot, dir);
    };
    for (int b = 0; b < nb; ++b) {
      lp.mass[b] = ld_par(pm.body[b][0], W.mass[b]);
      for (int c = 0; c < 3; ++c) lp.size[b][c] = ld_par(pm.body[b][c + 1], W.p[b][c]);
    }
    lp.friction = ld_par(pm.friction, W.friction);
    lp.restitution = ld_par(pm.restitution, W.restitution);
  }
  auto mass_of = [&](int b) -> T {
    if constexpr (PAR) return lp.mass[b];
    else return T(W.mass[b]);
  };
  auto size_of = [&](int b, int c) -> T {   // sphere radius (c = 0); capsule radius, length; box extents
    if constexpr (PAR) return lp.size[b][c];
    else return T(W.p[b][c]);
  };
  auto half_length = [&](int b) -> T {      // capsule half axis (0.5 L is exact: both forms give the same value)
    if constexpr (PAR) return T(0.5) * lp.size[b][1];
    else return T(0.5 * W.p[b][1]);
  };
  auto friction_of = [&]() -> T {
    if constexpr (PAR) return lp.friction;
    else return T(W.friction);
  };
  auto restitution_of = [&]() -> T {
    if constexpr (PAR) return lp.restitution;
    else return T(W.restitution);
  };
  V3<T> pos[TDS_RIGID_MAX_BODIES], lin[TDS_RIGID_MAX_BODIES], ang[TDS_RIGID_MAX_BODIES];
  T qx[TDS_RIGID_MAX_BODIES], qy[TDS_RIGID_MAX_BODIES], qz[TDS_RIGID_MAX_BODIES], qw[TDS_RIGID_MAX_BODIES];
  // input directions: the 13 * n_bodies state entries, then the 3 * n_bodies force entries
  for (int b = 0; b < nb; ++b) {
    auto ld = [&](int k) { return seed(T(s_in[(size_t)(b * 13 + k) * ns + e]), b * 13 + k); };
    pos[b] = v3<T>(ld(0), ld(1), ld(2));
    qx[b] = ld(3); qy[b] = ld(4); qz[b] = ld(5); qw[b] = ld(6);
    lin[b] = v3<T>(ld(7), ld(8), ld(9));
    ang[b] = v3<T>(ld(10), ld(11), ld(12));
  }
  const T dt = T(W.dt);
  Contact<T> cs[TDS_RIGID_MAX_CONTACTS];
  for (int s = 0; s < steps; ++s) {
    // apply_gravity, apply_force_impulse, clear_forces (rigid_body.hpp:84-101; the torque is always zero on this path)
    for (int b = 0; b < nb; ++b) {
      const T m = mass_of(b);
      const T inv_m = W.mass[b] == 0.0 ? T(0) : T(1) / m;
      V3<T> f = v3<T>(m * T(W.gravity[0]), m * T(W.gravity[1]), m * T(W.gravity[2]));
      if (s == 0 && force) {
        const int f0 = 13 * nb + 3 * b;
        f = f + v3<T>(seed(T(force[(size_t)(3 * b) * ns + e]), f0), seed(T(force[(size_t)(3 * b + 1) * ns + e]), f0 + 1),
                      seed(T(force[(size_t)(3 * b + 2) * ns + e]), f0 + 2));
      }
      lin[b] = lin[b] + f * inv_m * dt;
    }
    // contacts of every pair i < j (world.hpp:166-195)
    int nc = 0;
    for (int i = 0; i < nb; ++i)
      for (int j = i + 1; j < nb; ++j) {
        int a = i, b = j;
        int ta = W.type[a], tb = W.type[b];
        // direct function f[ta][tb], else the swapped one f[tb][ta] with points exchanged and normal negated
        const bool direct = (ta == TDSG_SPHERE && tb == TDSG_SPHERE) || (ta == TDSG_PLANE && (tb == TDSG_SPHERE || tb == TDSG_CAPSULE || tb == TDSG_BOX)) ||
                            (ta == TDSG_CAPSULE && tb == TDSG_SPHERE);
        const bool swapped = !direct && ((tb == TDSG_PLANE && (ta == TDSG_SPHERE || ta == TDSG_CAPSULE || ta == TDSG_BOX)) || (tb == TDSG_CAPSULE && ta == TDSG_SPHERE));
        if (!direct && !swapped) continue;
        if (swapped) { a = j; b = i; ta = W.type[a]; tb = W.type[b]; }     // the function runs on (a, b) = (j, i)
        const M3<T> Rb = quat_to_matrix<T>(qx[b], qy[b], qz[b], qw[b]);
        if (ta == TDSG_SPHERE) {
          sphere_sphere(pos[a], size_of(a, 0), pos[b], size_of(b, 0), cs, nc, a, b, pos[a], pos[b], swapped);
        } else if (ta == TDSG_CAPSULE) {   // contact_capsule_sphere: end spheres at +L/2, then -L/2
          const M3<T> Ra = quat_to_matrix<T>(qx[a], qy[a], qz[a], qw[a]);
          const V3<T> half = mul(Ra, v3<T>(T(0), T(0), half_length(a)));
          sphere_sphere(pos[a] + half, size_of(a, 0), pos[b], size_of(b, 0), cs, nc, a, b, pos[a], pos[b], swapped);
          sphere_sphere(pos[a] - half, size_of(a, 0), pos[b], size_of(b, 0), cs, nc, a, b, pos[a], pos[b], swapped);
        } else {                           // plane x sphere / capsule / box
          const V3<T> pn = v3<T>(T(W.p[a][0]), T(W.p[a][1]), T(W.p[a][2]));
          const T pc = T(W.p[a][3]);
          if (tb == TDSG_SPHERE) plane_sphere(pn, pc, pos[b], size_of(b, 0), cs, nc, a, b, pos[a], pos[b], swapped);
          else if (tb == TDSG_CAPSULE) {
            const V3<T> half = mul(Rb, v3<T>(T(0), T(0), half_length(b)));
            plane_sphere(pn, pc, pos[b] + half, size_of(b, 0), cs, nc, a, b, pos[a], pos[b], swapped);
            plane_sphere(pn, pc, pos[b] - half, size_of(b, 0), cs, nc, a, b, pos[a], pos[b], swapped);
          } else if constexpr (PAR) {      // as below, with the lane's extents
            const double r = 1e-2;
            const T dx = T(0.5) * lp.size[b][0] - T(r), dy = T(0.5) * lp.size[b][1] - T(r), dz = T(0.5) * lp.size[b][2] - T(r);
            for (int k = 0; k < 8; ++k) {
              const V3<T> corner = v3<T>((k & 4) ? -dx : dx, (k & 2) ? -dy : dy, (k & 1) ? -dz : dz);
              plane_sphere(pn, pc, pos[b] + mul(Rb, corner), T(r), cs, nc, a, b, pos[a], pos[b], swapped);
            }
          } else {                         // contact_plane_box: spheres of radius max(1e-2, 0) at the corners, x outermost
            const double r = 1e-2;
            const double dx = 0.5 * W.p[b][0] - r, dy = 0.5 * W.p[b][1] - r, dz = 0.5 * W.p[b][2] - r;
            for (int k = 0; k < 8; ++k) {
              const V3<T> corner = v3<T>(T((k & 4) ? -dx : dx), T((k & 2) ? -dy : dy), T((k & 1) ? -dz : dz));
              plane_sphere(pn, pc, pos[b] + mul(Rb, corner), T(r), cs, nc, a, b, pos[a], pos[b], swapped);
            }
          }
        }
      }
    // sequential impulses (world.hpp:336-340, rb_constraint_solver.hpp:113-160)
    for (int it = 0; it < W.num_solver_iterations; ++it)
      for (int c = 0; c < nc; ++c) {
        const Contact<T>& k = cs[c];
        if (!(k.dist < T(0))) continue;
        const int a = k.a, b = k.b;
        const T ima = W.mass[a] == 0.0 ? T(0) : T(1) / mass_of(a), imb = W.mass[b] == 0.0 ? T(0) : T(1) / mass_of(b);
        const T iia = W.mass[a] == 0.0 ? T(0) : T(1), iib = W.mass[b] == 0.0 ? T(0) : T(1);   // inv_inertia_world_: identity or zero (rigid_body.hpp:53-54)
        const T baumgarte = T(W.erp) * k.dist / dt;
        const V3<T> rel_vel = (lin[a] + cross(ang[a], k.ra)) - (lin[b] + cross(ang[b], k.rb));
        const T nrv = dot(k.n, rel_vel);
        if (!(nrv < T(0))) continue;
        const V3<T> t1 = cross(k.ra, k.n) * iia, t2 = cross(k.rb, k.n) * iib;
        const T angt = dot(k.n, cross(t1, k.ra) + cross(t2, k.rb));
        const T den = ima + imb + angt;
        const T impulse = (-(T(1) + restitution_of()) * nrv - baumgarte) / den;
        if (!(impulse > T(0))) continue;
        auto apply = [&](int body, const V3<T>& imp, const V3<T>& r, T im, T ii) {   // RigidBody::apply_impulse
          lin[body] = lin[body] + imp * im;
          ang[body] = ang[body] + cross(r, imp) * ii;
        };
        const V3<T> iv = k.n * impulse;
        apply(a, iv, k.ra, ima, iia);
        apply(b, v3<T>(-iv.x, -iv.y, -iv.z), k.rb, imb, iib);
        const V3<T> lat = rel_vel - k.n * nrv;             // (rel_vel from BEFORE the normal impulse, as the reference)
        const T lat_n = sqrt_t(dot(lat, lat));
        const T trial = lat_n / den;
        const T fi = trial < friction_of() * impulse ? trial : friction_of() * impulse;
        if (lat_n > T(1e-4)) {
          const V3<T> fd = lat * (T(1) / lat_n);
          apply(a, fd * (-fi), k.ra, ima, iia);
          apply(b, fd * fi, k.rb, imb, iib);
        }
      }
    // integrate (rigid_body.hpp:110-118; quat_velocity, tiny_algebra.hpp:604-614)
    for (int b = 0; b < nb; ++b) {
      pos[b] = pos[b] + lin[b] * dt;
      const T h = T(0.5) * dt;
      const V3<T> w = ang[b];
      const T dw = (-qx[b] * w.x - qy[b] * w.y - qz[b] * w.z) * h;
      const T dx = (qw[b] * w.x + qz[b] * w.y - qy[b] * w.z) * h;
      const T dy = (qw[b] * w.y + qx[b] * w.z - qz[b] * w.x) * h;
      const T dz = (qw[b] * w.z + qy[b] * w.x - qx[b] * w.y) * h;
      T x = qx[b] + dx, y = qy[b] + dy, z = qz[b] + dz, ww = qw[b] + dw;
      const T inv = T(1) / sqrt_t(x * x + y * y + z * z + ww * ww);
      qx[b] = x * inv; qy[b] = y * inv; qz[b] = z * inv; qw[b] = ww * inv;
    }
  }
  if constexpr (TP) {
    auto entry = [&](int r) -> T {   // state row r = 13 b + k
      const int b = r / 13, k = r % 13;
      switch (k) {
        case 0: return pos[b].x; case 1: return pos[b].y; case 2: return pos[b].z;
        case 3: return qx[b]; case 4: return qy[b]; case 5: return qz[b]; case 6: return qw[b];
        case 7: return lin[b].x; case 8: return lin[b].y; case 9: return lin[b].z;
        case 10: return ang[b].x; case 11: return ang[b].y; default: return ang[b].z;
      }
    };
    if constexpr (PAR) {
      if (vio.g_out) {
        double* adj = vio.adj + ((size_t)(e >> 5) * vio.cap * 32 + (e & 31));
        if (tape_reverse(adj, 13 * nb, [&](int r) { return entry(r).id; }, [&](int r) { return vio.g_out[(size_t)r * ns + e]; }, 16 * nb + pm.n)) {
          for (int r = 0; r < 13 * nb; ++r) vio.g_state[(size_t)r * ns + e] = adj[(size_t)r * 32];
          if (vio.g_force) for (int r = 0; r < 3 * nb; ++r) vio.g_force[(size_t)r * ns + e] = adj[(size_t)(13 * nb + r) * 32];
          if (pm.grad) for (int s = 0; s < pm.n; ++s) pm.grad[(size_t)s * ns + e] = adj[(size_t)(16 * nb + s) * 32];
        }
      }
    } else if (vio.g_out) {
      double* adj = vio.adj + ((size_t)(e >> 5) * vio.cap * 32 + (e & 31));
      if (tape_reverse(adj, 13 * nb, [&](int r) { return entry(r).id; }, [&](int r) { return vio.g_out[(size_t)r * ns + e]; }, 16 * nb)) {
        for (int r = 0; r < 13 * nb; ++r) vio.g_state[(size_t)r * ns + e] = adj[(size_t)r * 32];
        if (vio.g_force) for (int r = 0; r < 3 * nb; ++r) vio.g_force[(size_t)r * ns + e] = adj[(size_t)(13 * nb + r) * 32];
      }
    }
    if (s_out) for (int r = 0; r < 13 * nb; ++r) s_out[(size_t)r * ns + e] = (TS)val_of(entry(r));
    return;
  }
  for (int b = 0; b < nb; ++b) {
    const T out[13] = {pos[b].x, pos[b].y, pos[b].z, qx[b], qy[b], qz[b], qw[b], lin[b].x, lin[b].y, lin[b].z, ang[b].x, ang[b].y, ang[b].z};
    for (int k = 0; k < 13; ++k) {
      if constexpr (AD) {
        if constexpr (JV) vio.t_out[((size_t)(b * 13 + k) * vio.m + dir) * ns + e] = out[k].d;   // [row][tangent][world]
        else if constexpr (PAR) {   // parameter directions: column s of [row][k][world]; input directions as below
          if (jac) {
            if (dir >= 16 * nb) jac[((size_t)(b * 13 + k) * pm.n + (dir - 16 * nb)) * ns + e] = out[k].d;
            else jac[((size_t)(b * 13 + k) * (16 * nb) + dir) * ns + e] = out[k].d;
          }
        } else if (jac) jac[((size_t)(b * 13 + k) * (16 * nb) + dir) * ns + e] = out[k].d;     // [row][column][world]
        if (blockIdx.y == 0 && s_out) s_out[(size_t)(b * 13 + k) * ns + e] = (TS)val_of(out[k]);
      } else if constexpr (!TP) {
        s_out[(size_t)(b * 13 + k) * ns + e] = (TS)out[k];
      }
    }
  }
}
}  // namespace tdsrb

#ifndef TDS_RIGID_KERNEL_ONLY   // (tests/cpp/rigid_host.cpp compiles the kernel above for the host)
#include <string>
#include <vector>

#include "tds_host_io.h"

extern "C" void tds_b200_set_error(const char* msg);
// the PAR instances (csrc/tds_rigid_par.cu)
extern "C" int tds_launch_rigid_step_par(const RigidWorld* W, const RigidParMap* pm, const double* s_in, double* s_out, const double* force,
                                         int steps, int n, int ns, cudaStream_t stream);
extern "C" int tds_launch_rigid_jacobian_par(const RigidWorld* W, const RigidParMap* pm, const double* s_in, double* s_out, const double* force,
                                             int steps, int n, int ns, double* jac, int dir0, int n_dirs, cudaStream_t stream);
extern "C" int tds_launch_rigid_jvp_par(const RigidWorld* W, const RigidParMap* pm, const double* s_in, double* s_out, const double* force,
                                        int steps, int n, int ns, const tdsrb::RigidJvpIO* v, cudaStream_t stream);
extern "C" int tds_launch_rigid_vjp_par(const RigidWorld* W, const RigidParMap* pm, const double* s_in, double* s_out, const double* force,
                                        int n, int ns, const tdsrb::RigidVjpIO* v, cudaStream_t stream);
extern "C" int tds_launch_rigid_accumulate(double* dst, const double* src, int k, int n, int ns, cudaStream_t stream);

struct tds_b200_rigid {
  RigidWorld W;
  // installed physical parameters (par.n = 0: none; the map's pointers are set per launch).  par_dev [3][k][ns]: the values, the
  // staging of one reverse launch's parameter cotangents, g_par of the host path; it grows and is kept for new values
  RigidParMap par{};
  double* par_dev = nullptr; size_t par_bytes = 0;
  int n = 0, ns = 0, device = 0;
  double *state = nullptr, *state2 = nullptr, *force = nullptr, *jac = nullptr;   // state2: output of the differentiable instance
  size_t state2_bytes = 0, jac_bytes = 0;
  // vector-Jacobian product: checkpointed states, tape capacity (nodes per lane; doubles on overflow and stays grown), tape +
  // adjoint buffer, overflow flag, device staging of the host path
  double* ckpt = nullptr; size_t ckpt_bytes = 0;
  int tape_cap = 4096;
  char* vjp_buf = nullptr; size_t vjp_buf_bytes = 0;
  int* vjp_flag = nullptr;
  double* vjp_g = nullptr; size_t vjp_g_bytes = 0;   // [2 * 13 n_bodies + 3 n_bodies][ns]: g_state | next state cotangent | g_force of the host path
  double* jvp_buf = nullptr; size_t jvp_buf_bytes = 0;   // Jacobian-vector product, host path: t_state | t_force | t_state_out
  cudaStream_t stream = nullptr;
};

static int rigid_fail(const std::string& m, int rc) { tds_b200_set_error(m.c_str()); return rc; }
#define RB_TRY(expr) do { cudaError_t e_ = (expr); if (e_ != cudaSuccess) return rigid_fail(std::string(#expr) + ": " + cudaGetErrorString(e_), (int)e_); } while (0)

extern "C" {
// desc: [n_bodies][6] = mass, shape (TDSG_*), p0, p1, p2, p3 (see RigidWorld::p).  NULL on a refused description / no GPU.
tds_b200_rigid* tds_b200_rigid_create(const double* desc, int n_bodies, int n_worlds, int device) {
  if (!desc || n_bodies < 1 || n_bodies > TDS_RIGID_MAX_BODIES || n_worlds < 1) { tds_b200_set_error("rigid world: 1..16 bodies, >= 1 world"); return nullptr; }
  RigidWorld W0;
  const int rcw = tds_rigid_world_from_desc(desc, n_bodies, &W0);
  if (rcw == -1) { tds_b200_set_error("rigid world: shapes are sphere, plane, capsule, box"); return nullptr; }
  if (rcw == -2) { tds_b200_set_error("rigid world: more than 48 candidate contact points"); return nullptr; }
  if (cudaSetDevice(device) != cudaSuccess) { tds_b200_set_error("cudaSetDevice failed"); return nullptr; }
  tds_b200_rigid* h = new tds_b200_rigid;
  h->W = W0;
  h->n = n_worlds; h->ns = (n_worlds + 31) & ~31; h->device = device;
  if (cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess ||
      cudaMalloc((void**)&h->state, sizeof(double) * 13 * n_bodies * h->ns) != cudaSuccess ||
      cudaMalloc((void**)&h->force, sizeof(double) * 3 * n_bodies * h->ns) != cudaSuccess) {
    tds_b200_set_error("rigid world: allocation failed");
    cudaFree(h->state); cudaFree(h->force); if (h->stream) cudaStreamDestroy(h->stream);
    delete h;
    return nullptr;
  }
  return h;
}

void tds_b200_rigid_destroy(tds_b200_rigid* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  cudaFree(h->state); cudaFree(h->state2); cudaFree(h->force); cudaFree(h->jac);
  cudaFree(h->ckpt); cudaFree(h->vjp_buf); cudaFree(h->vjp_flag); cudaFree(h->vjp_g); cudaFree(h->jvp_buf); cudaFree(h->par_dev);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;
}

int tds_b200_rigid_set_params(tds_b200_rigid* h, double dt, const double* gravity, double friction, double restitution, double erp,
                              int num_solver_iterations) {
  if (!h || !gravity || !(dt > 0) || num_solver_iterations < 0) return rigid_fail("rigid_set_params: bad argument", -1);
  h->W.dt = dt; for (int k = 0; k < 3; ++k) h->W.gravity[k] = gravity[k];
  h->W.friction = friction; h->W.restitution = restitution; h->W.erp = erp; h->W.num_solver_iterations = num_solver_iterations;
  return 0;
}

int tds_b200_rigid_param_count(const tds_b200_rigid* h) { return h ? 2 + 4 * h->W.n_bodies : -1; }

// values: device [k][ns] (copied on `stream`, unchecked) or host [n][k] (checked, synchronous)
static int rigid_set_physical_params(tds_b200_rigid* h, int k, const int* ids, const double* values, bool device, void* stream) {
  const char* what = device ? "rigid_set_physical_params_device" : "rigid_set_physical_params_host";
  if (!h || k < 0 || (k > 0 && (!ids || !values))) return rigid_fail(std::string(what) + ": bad argument", -1);
  RigidParMap pm;
  if (const char* err = tds_rigid_par_map(h->W, k, ids, &pm)) return rigid_fail(std::string(what) + ": " + err, -2);
  if (!device)
    for (int e = 0; e < h->n; ++e)
      for (int s = 0; s < k; ++s)
        if (!tds_rigid_par_value_ok(ids[s], values[(size_t)e * k + s]))
          return rigid_fail(std::string(what) + ": values must be finite, masses and sizes > 0, friction and restitution >= 0", -3);
  RB_TRY(cudaSetDevice(h->device));
  if (k == 0) { h->par = pm; return 0; }
  const size_t sec = (size_t)k * h->ns, bytes = sizeof(double) * 3 * sec;
  if (bytes > h->par_bytes) {
    RB_TRY(cudaDeviceSynchronize());
    h->par.n = 0;
    RB_TRY(grow_dev(&h->par_dev, &h->par_bytes, bytes));
    RB_TRY(cudaMemset(h->par_dev, 0, bytes));
  }
  if (device) {
    RB_TRY(cudaMemcpyAsync(h->par_dev, values, sizeof(double) * sec, cudaMemcpyDeviceToDevice, stream ? (cudaStream_t)stream : h->stream));
  } else {
    // steps run on non-blocking streams, which this copy does not wait for
    RB_TRY(cudaDeviceSynchronize());
    RB_TRY(put_rows(h->par_dev, values, k, h->n, h->ns, h->stream));
    // a copy from pageable memory may return before its DMA has landed, and the non-blocking streams do not wait for it either
    RB_TRY(cudaDeviceSynchronize());
  }
  h->par = pm;
  return 0;
}

int tds_b200_rigid_set_physical_params_device(tds_b200_rigid* h, int k, const int* ids, const double* values, void* stream) {
  return rigid_set_physical_params(h, k, ids, values, true, stream);
}

int tds_b200_rigid_set_physical_params_host(tds_b200_rigid* h, int k, const int* ids, const double* values) {
  return rigid_set_physical_params(h, k, ids, values, false, nullptr);
}

// the installed map with its values for a launch over all worlds
static RigidParMap rigid_launch_map(const tds_b200_rigid* h) {
  RigidParMap pm = h->par;
  pm.values = h->par_dev; pm.t_par = nullptr; pm.grad = nullptr;
  return pm;
}

static int rigid_launch_rc(int err, const char* what) {
  return err ? rigid_fail(std::string(what) + ": " + cudaGetErrorString((cudaError_t)err), err) : 0;
}

// `steps` calls of World::step on device arrays [13 * n_bodies][n_stride] fp64 (n_stride = n_worlds rounded up to 32); force
// [3 * n_bodies][n_stride] or NULL = RigidBody::apply_central_force before the first step (forces are cleared by every step).
int tds_b200_rigid_step_device(tds_b200_rigid* h, const double* state_in, double* state_out, const double* force, int steps, void* stream) {
  if (!h || !state_in || !state_out || steps < 0) return rigid_fail("rigid_step_device: bad argument", -1);
  if (h->par.n) {
    const RigidParMap pm = rigid_launch_map(h);
    return rigid_launch_rc(tds_launch_rigid_step_par(&h->W, &pm, state_in, state_out, force, steps, h->n, h->ns,
                                                     stream ? (cudaStream_t)stream : h->stream), "rigid_step_device");
  }
  const int T = 128, B = (h->n + T - 1) / T;
  tdsrb::tds_rigid_step_kernel<double, double><<<B, T, 0, stream ? (cudaStream_t)stream : h->stream>>>(h->W, state_in, state_out, force, steps, h->n, h->ns, nullptr, 0);
  RB_TRY(cudaGetLastError());
  return 0;
}

// host state [n][13 nb] and force [n][3 nb] (or NULL) -> h->state, h->force
static int rigid_upload(tds_b200_rigid* h, const double* state, const double* force) {
  const int nb = h->W.n_bodies, n = h->n, ns = h->ns;
  RB_TRY(put_rows(h->state, state, 13 * nb, n, ns, h->stream));
  if (ns > n) {   // padding worlds hold the identity orientation: w (row 13 b + 6) = 1
    const std::vector<double> one((size_t)nb * (ns - n), 1.0);
    RB_TRY(cudaMemcpy2DAsync(h->state + (size_t)6 * ns + n, sizeof(double) * 13 * ns, one.data(), sizeof(double) * (ns - n),
                             sizeof(double) * (ns - n), nb, cudaMemcpyHostToDevice, h->stream));
    RB_TRY(cudaStreamSynchronize(h->stream));
  }
  if (force) RB_TRY(put_rows(h->force, force, 3 * nb, n, ns, h->stream));
  return 0;
}

// host arrays: state [n_worlds][n_bodies][13], force [n_worlds][n_bodies][3] or NULL, state_out like state
int tds_b200_rigid_step_host(tds_b200_rigid* h, const double* state, const double* force, int steps, double* state_out) {
  if (!h || !state || !state_out) return rigid_fail("rigid_step_host: bad argument", -1);
  RB_TRY(cudaSetDevice(h->device));
  int rc = rigid_upload(h, state, force);
  if (!rc) rc = tds_b200_rigid_step_device(h, h->state, h->state, force ? h->force : nullptr, steps, h->stream);
  if (rc) return rc;
  RB_TRY(get_rows(state_out, h->state, 13 * h->W.n_bodies, h->n, h->ns, h->stream));
  return 0;
}

// d state_out / d (state_in | force) by forward-mode dual numbers, one lane per (world, input direction):
// jac [n_worlds][13 * n_bodies][16 * n_bodies] (the billiard gradients of the reference's python/examples/billiard_optimization.py)
// params: over the installed parameters instead (jac [n_worlds][13 n_bodies][k])
static int rigid_jacobian(tds_b200_rigid* h, const double* state, const double* force, int steps, double* state_out, double* jac, bool params) {
  RB_TRY(cudaSetDevice(h->device));
  RB_TRY(cudaDeviceSynchronize());   // (device calls of this world on other streams may still use its derivative buffers)
  const int nb = h->W.n_bodies, n = h->n, ns = h->ns, rows = 13 * nb, cols = params ? h->par.n : 16 * nb;
  std::vector<double> zero_f;
  if (!force) { zero_f.assign((size_t)n * 3 * nb, 0.0); force = zero_f.data(); }
  int rc = rigid_upload(h, state, force);
  if (rc) return rc;
  // (sized for the 16 n_bodies input columns, which bound the k <= 2 + 4 n_bodies parameter columns)
  RB_TRY(grow_dev(&h->jac, &h->jac_bytes, sizeof(double) * (size_t)rows * 16 * nb * ns));
  RB_TRY(grow_dev(&h->state2, &h->state2_bytes, sizeof(double) * (size_t)rows * ns));   // (the lanes of other directions still read the input)
  if (h->par.n) {
    const RigidParMap pm = rigid_launch_map(h);
    rc = rigid_launch_rc(tds_launch_rigid_jacobian_par(&h->W, &pm, h->state, h->state2, h->force, steps, n, ns, h->jac, params ? 16 * nb : 0, cols,
                                                       h->stream), "rigid_jacobian");
    if (rc) return rc;
  } else {
    const int T = 128;
    dim3 grid((n + T - 1) / T, cols);
    tdsrb::tds_rigid_step_kernel<tds::Dual<double>, double><<<grid, T, 0, h->stream>>>(h->W, h->state, h->state2, h->force, steps, n, ns, h->jac, 0);
    RB_TRY(cudaGetLastError());
  }
  RB_TRY(get_rows(jac, h->jac, (size_t)rows * cols, n, ns, h->stream));
  if (state_out) RB_TRY(get_rows(state_out, h->state2, rows, n, ns, h->stream));
  return 0;
}

int tds_b200_rigid_jacobian_host(tds_b200_rigid* h, const double* state, const double* force, int steps, double* state_out, double* jac) {
  if (!h || !state || !jac) return rigid_fail("rigid_jacobian_host: bad argument", -1);
  return rigid_jacobian(h, state, force, steps, state_out, jac, false);
}

int tds_b200_rigid_param_jacobian_host(tds_b200_rigid* h, const double* state, const double* force, int steps, double* state_out, double* jac) {
  if (!h || !state || !jac || steps < 0) return rigid_fail("rigid_param_jacobian_host: bad argument", -1);
  if (!h->par.n) return rigid_fail("rigid_param_jacobian_host: no physical parameters installed", -4);
  return rigid_jacobian(h, state, force, steps, state_out, jac, true);
}

using tdsrb::RigidVjpIO;
using tds::Tape;
using tds::TapeNode;

// One launch of the taping instance over every world, in chunks of worlds whose tape + adjoints stay inside 2 GB; a chunk whose
// tape overflowed is rerun with twice the capacity.  vio: g_out / g_state / g_force for all worlds (offset per chunk here).  With
// installed parameters the PAR instance runs; g_par [k][ns] (or null) then receives the sum of the parameter cotangents of the
// recorded step: a chunk writes them to the staging section of par_dev, which is added to g_par only once the chunk's overflow
// flag reads clear, so a rerun chunk is never counted twice.
static int rigid_tape_pass(tds_b200_rigid* h, const double* s_in, double* s_out, const double* force, RigidVjpIO vio, cudaStream_t sm,
                           double* g_par = nullptr) {
  const int n = h->n, ns = h->ns;
  if (!h->vjp_flag) RB_TRY(cudaMalloc((void**)&h->vjp_flag, sizeof(int)));
  const bool record = vio.g_out != nullptr;
  for (int e0 = 0; e0 < n;) {
    const size_t lane_bytes = record ? (size_t)h->tape_cap * (sizeof(TapeNode) + sizeof(double)) : 0;
    size_t warps = record ? (((size_t)2 << 30) / (32 * lane_bytes)) : (size_t)(n + 31) / 32;
    if (warps < 1) warps = 1;
    const size_t left = (size_t)(n - e0 + 31) / 32;
    if (warps > left) warps = left;
    const int chunk = (int)(warps * 32 < (size_t)(n - e0) ? warps * 32 : (size_t)(n - e0));
    const size_t tape_b = warps * 32 * h->tape_cap * sizeof(TapeNode), need = record ? warps * 32 * lane_bytes : 0;
    if (need > h->vjp_buf_bytes) RB_TRY(cudaStreamSynchronize(sm));   // (earlier chunks still use the buffer)
    RB_TRY(grow_dev(&h->vjp_buf, &h->vjp_buf_bytes, need));
    RigidVjpIO v = vio;
    if (record) {
      v.g_out += e0; v.g_state += e0; if (v.g_force) v.g_force += e0;
      v.tape = (TapeNode*)h->vjp_buf; v.adj = (double*)(h->vjp_buf + tape_b); v.cap = h->tape_cap; v.overflow = h->vjp_flag;
      RB_TRY(cudaMemsetAsync(h->vjp_flag, 0, sizeof(int), sm));
    }
    double* stage = h->par.n ? h->par_dev + (size_t)h->par.n * ns : nullptr;
    if (h->par.n) {
      RigidParMap pm = rigid_launch_map(h);
      pm.values += e0;
      pm.grad = record && g_par ? stage + e0 : nullptr;
      const int rc = rigid_launch_rc(tds_launch_rigid_vjp_par(&h->W, &pm, s_in + e0, s_out ? s_out + e0 : nullptr, force ? force + e0 : nullptr,
                                                              chunk, ns, &v, sm), "rigid_vjp");
      if (rc) return rc;
    } else {
      const int T = 128, B = (chunk + T - 1) / T;
      tdsrb::tds_rigid_step_kernel<Tape<double>, double><<<B, T, 0, sm>>>(h->W, s_in + e0, s_out ? s_out + e0 : nullptr,
                                                                          force ? force + e0 : nullptr, 1, chunk, ns, nullptr, 0, v);
      RB_TRY(cudaGetLastError());
    }
    if (record) {
      int overflow = 0;
      RB_TRY(cudaMemcpyAsync(&overflow, h->vjp_flag, sizeof(int), cudaMemcpyDeviceToHost, sm));
      RB_TRY(cudaStreamSynchronize(sm));
      if (overflow) {
        if (h->tape_cap > (1 << 28)) return rigid_fail("rigid_vjp: tape capacity exhausted", -4);
        h->tape_cap *= 2;
        continue;
      }
      if (g_par && h->par.n) {
        const int rc = rigid_launch_rc(tds_launch_rigid_accumulate(g_par + e0, stage + e0, h->par.n, chunk, ns, sm), "rigid_vjp");
        if (rc) return rc;
      }
    }
    e0 += chunk;
  }
  return 0;
}

// vjp_g, the state and force cotangents of the VJP: [2 * 13 n_bodies + 3 n_bodies][ns]
static cudaError_t grow_vjp_g(tds_b200_rigid* h) {
  return grow_dev(&h->vjp_g, &h->vjp_g_bytes, sizeof(double) * (size_t)(2 * 13 + 3) * h->W.n_bodies * h->ns);
}

// g_par: [k][ns] sum over the steps of the installed parameters' cotangents, or null
static int rigid_vjp(tds_b200_rigid* h, const double* state, const double* force, int steps, const double* g_state_out,
                     double* g_state, double* g_force, double* g_par, cudaStream_t sm) {
  const int nb = h->W.n_bodies, ns = h->ns, rows = 13 * nb;
  const size_t sb = sizeof(double) * (size_t)rows * ns;
  if (g_state != g_state_out) RB_TRY(cudaMemcpyAsync(g_state, g_state_out, sb, cudaMemcpyDeviceToDevice, sm));
  if (g_force) RB_TRY(cudaMemsetAsync(g_force, 0, sizeof(double) * 3 * nb * ns, sm));
  if (g_par) RB_TRY(cudaMemsetAsync(g_par, 0, sizeof(double) * h->par.n * ns, sm));
  if (steps == 0) return 0;
  // forward, one step at a time, by the same instance without recording: states 0 .. steps - 1 are kept
  if (sb * steps > h->ckpt_bytes) RB_TRY(cudaStreamSynchronize(sm));   // (the last call's work may still read the checkpoints)
  RB_TRY(grow_dev(&h->ckpt, &h->ckpt_bytes, sb * steps));
  RB_TRY(cudaMemcpyAsync(h->ckpt, state, sb, cudaMemcpyDeviceToDevice, sm));
  RB_TRY(grow_vjp_g(h));
  const size_t st = (size_t)rows * ns;
  for (int k = 0; k + 1 < steps; ++k) {
    int rc = rigid_tape_pass(h, h->ckpt + k * st, h->ckpt + (k + 1) * st, k == 0 ? force : nullptr, RigidVjpIO{}, sm);
    if (rc) return rc;
  }
  // reverse: one recorded step per launch, the state cotangent chained through g_state
  double* gnext = h->vjp_g == g_state ? h->vjp_g + st : h->vjp_g;   // (the host path passes its own staging as g_state)
  for (int k = steps - 1; k >= 0; --k) {
    RigidVjpIO v{};
    v.g_out = g_state; v.g_state = gnext; v.g_force = k == 0 ? g_force : nullptr;
    int rc = rigid_tape_pass(h, h->ckpt + k * st, nullptr, k == 0 ? force : nullptr, v, sm, g_par);
    if (rc) return rc;
    RB_TRY(cudaMemcpyAsync(g_state, gnext, sb, cudaMemcpyDeviceToDevice, sm));
  }
  return 0;
}

int tds_b200_rigid_vjp_device(tds_b200_rigid* h, const double* state, const double* force, int steps, const double* g_state_out,
                              double* g_state, double* g_force, void* stream) {
  if (!h || !state || !g_state_out || !g_state || steps < 0) return rigid_fail("rigid_vjp_device: bad argument", -1);
  return rigid_vjp(h, state, force, steps, g_state_out, g_state, g_force, nullptr, stream ? (cudaStream_t)stream : h->stream);
}

int tds_b200_rigid_vjp_params_device(tds_b200_rigid* h, const double* state, const double* force, int steps, const double* g_state_out,
                                     double* g_state, double* g_force, double* g_par, void* stream) {
  if (!h || !state || !g_state_out || !g_state || !g_par || steps < 0) return rigid_fail("rigid_vjp_params_device: bad argument", -1);
  if (!h->par.n) return rigid_fail("rigid_vjp_params_device: no physical parameters installed", -4);
  return rigid_vjp(h, state, force, steps, g_state_out, g_state, g_force, g_par, stream ? (cudaStream_t)stream : h->stream);
}

// host arrays; g_par [n][k] or null
static int rigid_vjp_host(tds_b200_rigid* h, const double* state, const double* force, int steps, const double* g_state_out,
                          double* g_state, double* g_force, double* g_par) {
  RB_TRY(cudaSetDevice(h->device));
  RB_TRY(cudaDeviceSynchronize());   // (device calls of this world on other streams may still use its derivative buffers)
  const int nb = h->W.n_bodies, n = h->n, ns = h->ns, rows = 13 * nb;
  int rc = rigid_upload(h, state, force);
  if (rc) return rc;
  RB_TRY(grow_vjp_g(h));
  double* gs = h->vjp_g;
  double* gf = h->vjp_g + (size_t)2 * rows * ns;
  double* gp = g_par ? h->par_dev + (size_t)2 * h->par.n * ns : nullptr;
  RB_TRY(put_rows(gs, g_state_out, rows, n, ns, h->stream));
  if ((rc = rigid_vjp(h, h->state, force ? h->force : nullptr, steps, gs, gs, gf, gp, h->stream))) return rc;
  RB_TRY(get_rows(g_state, gs, rows, n, ns, h->stream));
  if (g_force) RB_TRY(get_rows(g_force, gf, 3 * nb, n, ns, h->stream));
  if (gp) RB_TRY(get_rows(g_par, gp, h->par.n, n, ns, h->stream));
  return 0;
}

int tds_b200_rigid_vjp_host(tds_b200_rigid* h, const double* state, const double* force, int steps, const double* g_state_out,
                            double* g_state, double* g_force) {
  if (!h || !state || !g_state_out || !g_state || steps < 0) return rigid_fail("rigid_vjp_host: bad argument", -1);
  return rigid_vjp_host(h, state, force, steps, g_state_out, g_state, g_force, nullptr);
}

int tds_b200_rigid_vjp_params_host(tds_b200_rigid* h, const double* state, const double* force, int steps, const double* g_state_out,
                                   double* g_state, double* g_force, double* g_par) {
  if (!h || !state || !g_state_out || !g_state || !g_par || steps < 0) return rigid_fail("rigid_vjp_params_host: bad argument", -1);
  if (!h->par.n) return rigid_fail("rigid_vjp_params_host: no physical parameters installed", -4);
  return rigid_vjp_host(h, state, force, steps, g_state_out, g_state, g_force, g_par);
}

// Jacobian-vector products of `steps` steps: one launch of the tangent-seeded dual instance, one lane per (world, tangent), each lane
// runs the whole rollout.  A force tangent with a null force acts on a zero force (the handle's force buffer is cleared for it).
// With installed parameters the PAR instance runs, t_par [k * m][ns] (null: zero tangent).
static int rigid_jvp(tds_b200_rigid* h, const double* state, const double* force, int steps, int m, const double* t_state,
                     const double* t_force, const double* t_par, double* state_out, double* t_state_out, cudaStream_t sm) {
  const int nb = h->W.n_bodies;
  if (!force && t_force) {
    RB_TRY(cudaMemsetAsync(h->force, 0, sizeof(double) * 3 * nb * h->ns, sm));
    force = h->force;
  }
  const tdsrb::RigidJvpIO v{t_state, t_force, t_state_out, m};
  if (h->par.n) {
    RigidParMap pm = rigid_launch_map(h);
    pm.t_par = t_par;
    return rigid_launch_rc(tds_launch_rigid_jvp_par(&h->W, &pm, state, state_out, force, steps, h->n, h->ns, &v, sm), "rigid_jvp");
  }
  const int T = 128;
  const dim3 grid((h->n + T - 1) / T, m);
  tdsrb::tds_rigid_step_kernel<tds::Dual<double>, double, true><<<grid, T, 0, sm>>>(h->W, state, state_out, force, steps, h->n, h->ns,
                                                                                   nullptr, 0, v);
  RB_TRY(cudaGetLastError());
  return 0;
}

int tds_b200_rigid_jvp_device(tds_b200_rigid* h, const double* state, const double* force, int steps, int m, const double* t_state,
                              const double* t_force, double* state_out, double* t_state_out, void* stream) {
  if (!h || !state || !t_state_out || steps < 0 || m < 1 || m > 65535 || (!t_state && !t_force) || state_out == state)
    return rigid_fail("rigid_jvp_device: bad argument", -1);
  return rigid_jvp(h, state, force, steps, m, t_state, t_force, nullptr, state_out, t_state_out, stream ? (cudaStream_t)stream : h->stream);
}

int tds_b200_rigid_jvp_params_device(tds_b200_rigid* h, const double* state, const double* force, int steps, int m, const double* t_state,
                                     const double* t_force, const double* t_par, double* state_out, double* t_state_out, void* stream) {
  if (!h || !state || !t_state_out || steps < 0 || m < 1 || m > 65535 || (!t_state && !t_force && !t_par) || state_out == state)
    return rigid_fail("rigid_jvp_params_device: bad argument", -1);
  if (!h->par.n) return rigid_fail("rigid_jvp_params_device: no physical parameters installed", -4);
  return rigid_jvp(h, state, force, steps, m, t_state, t_force, t_par, state_out, t_state_out, stream ? (cudaStream_t)stream : h->stream);
}

// host arrays; t_par [n][k][m] or null
static int rigid_jvp_host(tds_b200_rigid* h, const double* state, const double* force, int steps, int m, const double* t_state,
                          const double* t_force, const double* t_par, double* state_out, double* t_state_out) {
  RB_TRY(cudaSetDevice(h->device));
  RB_TRY(cudaDeviceSynchronize());   // (device calls of this world on other streams may still use its derivative buffers)
  const int nb = h->W.n_bodies, n = h->n, ns = h->ns, rows = 13 * nb;
  int rc = rigid_upload(h, state, force);
  if (rc) return rc;
  // tangents: host [n][dim][m] <-> device [dim * m][ns]; t_state | t_force | t_state_out | t_par
  const size_t ts = (size_t)rows * m, tf = (size_t)3 * nb * m, tp = t_par ? (size_t)h->par.n * m : 0;
  RB_TRY(grow_dev(&h->jvp_buf, &h->jvp_buf_bytes, sizeof(double) * (2 * ts + tf + tp) * ns));
  RB_TRY(grow_dev(&h->state2, &h->state2_bytes, sizeof(double) * (size_t)rows * ns));
  double *ds = h->jvp_buf, *df = ds + ts * ns, *dout = df + tf * ns, *dp = dout + ts * ns;
  if (t_state) RB_TRY(put_rows(ds, t_state, ts, n, ns, h->stream));
  if (t_force) RB_TRY(put_rows(df, t_force, tf, n, ns, h->stream));
  if (t_par) RB_TRY(put_rows(dp, t_par, tp, n, ns, h->stream));
  rc = rigid_jvp(h, h->state, force ? h->force : nullptr, steps, m, t_state ? ds : nullptr, t_force ? df : nullptr, t_par ? dp : nullptr,
                 h->state2, dout, h->stream);
  if (rc) return rc;
  RB_TRY(get_rows(t_state_out, dout, ts, n, ns, h->stream));
  if (state_out) RB_TRY(get_rows(state_out, h->state2, rows, n, ns, h->stream));
  return 0;
}

int tds_b200_rigid_jvp_host(tds_b200_rigid* h, const double* state, const double* force, int steps, int m, const double* t_state,
                            const double* t_force, double* state_out, double* t_state_out) {
  if (!h || !state || !t_state_out || steps < 0 || m < 1 || m > 65535 || (!t_state && !t_force)) return rigid_fail("rigid_jvp_host: bad argument", -1);
  return rigid_jvp_host(h, state, force, steps, m, t_state, t_force, nullptr, state_out, t_state_out);
}

int tds_b200_rigid_jvp_params_host(tds_b200_rigid* h, const double* state, const double* force, int steps, int m, const double* t_state,
                                   const double* t_force, const double* t_par, double* state_out, double* t_state_out) {
  if (!h || !state || !t_state_out || steps < 0 || m < 1 || m > 65535 || (!t_state && !t_force && !t_par))
    return rigid_fail("rigid_jvp_params_host: bad argument", -1);
  if (!h->par.n) return rigid_fail("rigid_jvp_params_host: no physical parameters installed", -4);
  return rigid_jvp_host(h, state, force, steps, m, t_state, t_force, t_par, state_out, t_state_out);
}
}  // extern "C"
#endif  // TDS_RIGID_KERNEL_ONLY
