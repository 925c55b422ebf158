// C-ABI of libtds_b200.so (include/tds_b200.h): simulator lifecycle, device fast path, host-buffer
// paths and the reference's "C-ABI v1" drop-in symbols for the Laikago model.
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <mutex>
#include <string>
#include <vector>

#include "tds_b200.h"
#include "tds_b200_model.h"
#include "tds_model.h"
#include "tds_types.h"
#include "tds_team.h"
#include "tds_tape.cuh"
#include "tds_host_io.h"

extern "C" int tds_launch_stept(const TeamModel* TM, const TeamLink* tl_dev, const DevModel* M, const SimParams* P,
                                const EnvParams* E, const StepIO* io, int mode, int use_pd, int precision,
                                char* gscratch, int use_smem, cudaStream_t stream);
extern "C" size_t tds_stept_tile_bytes(const TeamModel* TM);
extern "C" unsigned long long tds_stepr_table_owner(int dev);
extern "C" int tds_launch_stepr(const TeamModel* TM, const TeamLink* tl_host, unsigned long long token, const DevModel* M,
                                const SimParams* P, const EnvParams* E, const StepIO* io, int mode, int use_pd,
                                int precision, char* gscratch, int use_smem, cudaStream_t stream);
extern "C" size_t tds_stepr_tile_bytes(const TeamModel* TM);
extern "C" int tds_spec_find(const double* model, int n_model, const DevModel* D, const EnvParams* E);
extern "C" size_t tds_spec_smem_bytes(int spec, int precision);
extern "C" const char* tds_spec_name(int spec);
extern "C" int tds_launch_step_spec(int spec, const SimParams* P, const EnvParams* E, const StepIO* io, int mode, int use_pd,
                                    int precision, cudaStream_t stream);
extern "C" int tds_launch_stepw_jacobian(const DevModel* M, const SimParams* P, const EnvParams* E, const StepIO* io, int mode,
                                         int use_pd, int n_dirs, char* gscratch, cudaStream_t stream);
extern "C" int tds_launch_stepw_vjp(const DevModel* M, const SimParams* P, const EnvParams* E, const StepIO* io, int mode,
                                    int use_pd, char* gscratch, cudaStream_t stream);
extern "C" int tds_launch_stepw(const DevModel* M, const SimParams* P, const EnvParams* E, const StepIO* io,
                                int mode, int use_pd, int precision, char* gscratch, int use_smem,
                                int warps_per_block, cudaStream_t stream);
// the same with installed physical parameters (tds_stepw_par.cu)
extern "C" int tds_launch_stepw_par(const DevModel* M, const SimParams* P, const EnvParams* E, const StepIO* io, const ParMap* pm,
                                    int mode, int use_pd, int precision, char* gscratch, int use_smem, int warps_per_block,
                                    cudaStream_t stream);
extern "C" int tds_launch_stepw_jacobian_par(const DevModel* M, const SimParams* P, const EnvParams* E, const StepIO* io, const ParMap* pm,
                                             int mode, int use_pd, int n_dirs, char* gscratch, cudaStream_t stream);
extern "C" int tds_launch_stepw_vjp_par(const DevModel* M, const SimParams* P, const EnvParams* E, const StepIO* io, const ParMap* pm,
                                        int mode, int use_pd, char* gscratch, cudaStream_t stream);
// Jacobian-vector products, with or without installed parameters (tds_stepw_jvp.cu)
extern "C" int tds_launch_stepw_jvp(const DevModel* M, const SimParams* P, const EnvParams* E, const StepIO* io, const ParMap* pm,
                                    const double* t_in, const double* t_par, int m, int mode, int use_pd, int n_dirs, char* gscratch,
                                    cudaStream_t stream);
// mass matrix M(q), its Jacobian-vector products and the two helper kernels of its vector-Jacobian product (tds_mass.cu)
extern "C" int tds_launch_mass(const DevModel* M, const StepIO* io, const ParMap* pm, char* gscratch, cudaStream_t stream);
extern "C" int tds_launch_mass_jvp(const DevModel* M, const StepIO* io, const ParMap* pm, const double* t_q, const double* t_par, int m,
                                   int n_dirs, char* gscratch, cudaStream_t stream);
extern "C" int tds_launch_mass_eye(double* t_q, double* t_par, int n_q, int k, int d0, int m, int ns, cudaStream_t stream);
extern "C" int tds_launch_mass_contract(const double* G, const double* dM, int nn, int m, int d0, int n_q, double* g_q, double* g_par, int n,
                                        int ns, cudaStream_t stream);
// forward kinematics and point Jacobians, and their Jacobian-vector products (tds_kin.cu)
extern "C" int tds_launch_kin(const DevModel* M, const StepIO* io, const TdsKinCall* kc, char* gscratch, cudaStream_t stream);
extern "C" int tds_launch_kin_jvp(const DevModel* M, const StepIO* io, const TdsKinCall* kc, const double* t_q, int m, int n_dirs,
                                  char* gscratch, cudaStream_t stream);
// inverse dynamics tau = ID(q, qd, qdd) and its Jacobian-vector products (tds_invdyn.cu)
extern "C" int tds_launch_inv(const DevModel* M, const SimParams* P, const StepIO* io, const ParMap* pm, char* gscratch, cudaStream_t stream);
extern "C" int tds_launch_inv_jvp(const DevModel* M, const SimParams* P, const StepIO* io, const ParMap* pm, const double* t_in,
                                  const double* t_par, int m, int n_dirs, char* gscratch, cudaStream_t stream);
// the step that reports its contacts, and its Jacobian-vector products (tds_contacts.cu)
extern "C" int tds_launch_contacts(const DevModel* M, const SimParams* P, const EnvParams* E, const StepIO* io, const ParMap* pm, float* cf,
                                   int mode, int use_pd, int precision, char* gscratch, cudaStream_t stream);
extern "C" int tds_launch_contacts_jvp(const DevModel* M, const SimParams* P, const EnvParams* E, const StepIO* io, const ParMap* pm,
                                       const double* t_in, const double* t_par, int m, int mode, int use_pd, int n_dirs, char* gscratch,
                                       cudaStream_t stream);
// the body record, centroidal momentum matrix and its bias, and their Jacobian-vector products (tds_centroidal.cu)
extern "C" int tds_launch_centroidal(const DevModel* M, const StepIO* io, const ParMap* pm, const TdsCenCall* out, char* gscratch,
                                     cudaStream_t stream);
extern "C" int tds_launch_centroidal_jvp(const DevModel* M, const StepIO* io, const ParMap* pm, const TdsCenCall* out, const double* t_in,
                                         const double* t_par, int m, int n_dirs, char* gscratch, cudaStream_t stream);
// the step with external wrenches, and its Jacobian-vector products (tds_wrench.cu)
extern "C" int tds_launch_wrench(const DevModel* M, const SimParams* P, const EnvParams* E, const StepIO* io, const ParMap* pm,
                                 const TdsExtCall* xc, int mode, int use_pd, int precision, char* gscratch, cudaStream_t stream);
extern "C" int tds_launch_wrench_jvp(const DevModel* M, const SimParams* P, const EnvParams* E, const StepIO* io, const ParMap* pm,
                                     const TdsExtCall* xc, const double* t_in, const double* t_par, int m, int mode, int use_pd, int n_dirs,
                                     char* gscratch, cudaStream_t stream);
// spatial point Jacobians, point velocities and accelerations, and their Jacobian-vector products (tds_point_motion.cu)
extern "C" int tds_launch_point_motion(const DevModel* M, const StepIO* io, const TdsMotCall* mc, char* gscratch, cudaStream_t stream);
extern "C" int tds_launch_point_motion_jvp(const DevModel* M, const StepIO* io, const TdsMotCall* mc, const double* t_in, int m, int n_dirs,
                                           char* gscratch, cudaStream_t stream);
// joint-torque and energy regressors of the inertial parameters, and their Jacobian-vector products (tds_regressor.cu)
extern "C" int tds_launch_regressor(const DevModel* M, const SimParams* P, const StepIO* io, const TdsRegCall* out, char* gscratch,
                                    cudaStream_t stream);
extern "C" int tds_launch_regressor_jvp(const DevModel* M, const SimParams* P, const StepIO* io, const TdsRegCall* out, const double* t_in,
                                        int m, int n_dirs, char* gscratch, cudaStream_t stream);
// inverse mass matrix M^-1(q), its Jacobian-vector products, and the contraction J M^-1 J^T (tds_mass_inverse.cu)
extern "C" int tds_launch_mass_inverse(const DevModel* M, const StepIO* io, const ParMap* pm, char* gscratch, cudaStream_t stream);
extern "C" int tds_launch_mass_inverse_jvp(const DevModel* M, const StepIO* io, const ParMap* pm, const double* t_q, const double* t_par,
                                           int m, int n_dirs, char* gscratch, cudaStream_t stream);
extern "C" int tds_launch_osim(const double* J, const double* dJ, const double* Mi, const double* dMi, double* L, int K, int n_qd, int m,
                               int n, int ns, cudaStream_t stream);
// Coriolis matrix C(q, qd) and its Jacobian-vector products (tds_coriolis.cu)
extern "C" int tds_launch_coriolis(const DevModel* M, const StepIO* io, const ParMap* pm, char* gscratch, cudaStream_t stream);
// Derivatives d tau / dq, d tau / dqd of the inverse dynamics and their Jacobian-vector products (tds_dynamics_derivatives.cu)
extern "C" int tds_launch_dynamics_derivatives(const DevModel* M, const SimParams* P, const StepIO* io, const ParMap* pm, char* gscratch,
                                               cudaStream_t stream);
extern "C" int tds_launch_dynamics_derivatives_jvp(const DevModel* M, const SimParams* P, const StepIO* io, const ParMap* pm, const double* t_in,
                                                   const double* t_par, int m, int n_dirs, char* gscratch, cudaStream_t stream);
extern "C" int tds_launch_coriolis_jvp(const DevModel* M, const StepIO* io, const ParMap* pm, const double* t_in, const double* t_par, int m,
                                       int n_dirs, char* gscratch, cudaStream_t stream);
// the rows and the solve of the point-constrained forward dynamics (tds_constrained.cu)
extern "C" int tds_launch_cdyn(const TdsCdynCall* c, int dual, int n, int ns, cudaStream_t stream);
// the product -M^-1 [d tau / dq | d tau / dqd] of the forward dynamics' derivatives (tds_fd_derivatives.cu)
extern "C" int tds_launch_fdd(const TdsFddCall* c, int dual, int n, int ns, cudaStream_t stream);
static_assert(TDS_B200_MAX_KIN_POINTS == TDS_MAX_KIN_POINTS, "the point table of the kernel argument holds the C-ABI's maximum");

// candidate contact points of a model, reference enumeration order: (link_a, link_b) per point
// (plane candidates first, then - worlds of several multibodies - the candidates between multibodies, list after list)
struct ContactCandTable {
  int n_points;
  signed char link_a[TDS_MAX_POINTS + TDS_MAX_PAIR_POINTS], link_b[TDS_MAX_POINTS + TDS_MAX_PAIR_POINTS];   // link index inside its multibody
  signed char body_a[TDS_MAX_POINTS + TDS_MAX_PAIR_POINTS], body_b[TDS_MAX_POINTS + TDS_MAX_PAIR_POINTS];   // multibody of the world (0 = the plane)
  signed char geom_a[TDS_MAX_POINTS + TDS_MAX_PAIR_POINTS], geom_b[TDS_MAX_POINTS + TDS_MAX_PAIR_POINTS];   // index in collision_geometries(link)
};

// Candidate points of a model in the reference's enumeration order (World::compute_contacts_multi_body_internal,
// src/world.hpp:212-281).  The plane is multibody 0 of the world, created first (body A of its contacts, base link -1); the
// multibodies of the model follow as 1, 2, ...; link indices are the reference's: inside their multibody.
static ContactCandTable make_cand_table(const DevModel& D) {
  ContactCandTable T;
  memset(&T, 0, sizeof(T));
  int first[TDS_MAX_LINKS + 1];   // first link of every multibody
  for (int i = 0, b = -1; i < D.n_links; ++i) if (D.body_of[i] != b) { b = D.body_of[i]; first[b] = i; }
  auto local = [&](int link) { return link < 0 ? -1 : link - first[D.body_of[link]]; };
  auto geom_in_link = [&](int g) { return g - D.geom_begin[D.g_link[g] + 1]; };   // iii / jjj of the reference's loops
  int c = 0;
  if (D.has_plane)
    for (int g = 0; g < D.n_geoms; ++g) {
      const int pts = D.g_type[g] == TDSG_SPHERE ? 1 : (D.g_type[g] == TDSG_CAPSULE ? 2 : (D.g_type[g] == TDSG_BOX ? 8 : 0));
      for (int j = 0; j < pts; ++j, ++c) {
        T.body_a[c] = 0; T.link_a[c] = -1; T.geom_a[c] = 0; T.geom_b[c] = (signed char)geom_in_link(g);
        T.body_b[c] = (signed char)(1 + (D.g_link[g] < 0 ? 0 : D.body_of[D.g_link[g]])); T.link_b[c] = (signed char)local(D.g_link[g]);
      }
    }
  for (int p = 0; p < D.n_pair_points; ++p, ++c) {
    const int la = D.g_link[D.pp_ga[p]], lb = D.g_link[D.pp_gb[p]];
    T.body_a[c] = (signed char)(1 + D.body_of[la]); T.link_a[c] = (signed char)local(la);
    T.body_b[c] = (signed char)(1 + D.body_of[lb]); T.link_b[c] = (signed char)local(lb);
    T.geom_a[c] = (signed char)geom_in_link(D.pp_ga[p]); T.geom_b[c] = (signed char)geom_in_link(D.pp_gb[p]);
  }
  T.n_points = c;
  return T;
}

namespace {

std::string g_err;  // mirror of the last error (the public accessor lives in urdf_model.cpp)
extern "C" void tds_b200_set_error(const char* msg);
void set_err(const std::string& s) { g_err = s; tds_b200_set_error(s.c_str()); }

#define CUDA_TRY(expr)                                                                  \
  do {                                                                                  \
    cudaError_t _e = (expr);                                                            \
    if (_e != cudaSuccess) {                                                            \
      set_err(std::string(#expr) + ": " + cudaGetErrorString(_e));                      \
      return (int)_e;                                                                   \
    }                                                                                   \
  } while (0)

// ---- layout conversion kernels (host AoS fp64/fp32 <-> device SoA fp32) --------------------------
template <typename TI>
__global__ void aos_to_soa_kernel(const TI* __restrict__ in, int in_stride, int in_off, float* __restrict__ out,
                                  int dim, int n, int ns) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  for (int k = 0; k < dim; ++k) out[(size_t)k * ns + e] = (float)in[(size_t)e * in_stride + in_off + k];
}
template <typename TO>
__global__ void soa_to_aos_kernel(const float* __restrict__ in, TO* __restrict__ out, int out_stride, int out_off,
                                  int dim, int n, int ns) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  for (int k = 0; k < dim; ++k) out[(size_t)e * out_stride + out_off + k] = (TO)in[(size_t)k * ns + e];
}

// obs[e] = q | qd (AoS), and optionally reward / done appended behind the n observation rows (one contiguous
// block -> one device->host copy when the caller's three output buffers are adjacent)
__global__ void pack_env_out_kernel(const float* __restrict__ q, const float* __restrict__ qd, const float* __restrict__ reward,
                                    const float* __restrict__ done, float* __restrict__ out, int n_q, int n_qd, int n, int ns,
                                    int with_tail) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  float* o = out + (size_t)e * (n_q + n_qd);
  for (int k = 0; k < n_q; ++k) o[k] = q[(size_t)k * ns + e];
  for (int k = 0; k < n_qd; ++k) o[n_q + k] = qd[(size_t)k * ns + e];
  if (with_tail) {
    float* tail = out + (size_t)n * (n_q + n_qd);
    tail[e] = reward[e];
    tail[n + e] = done[e];
  }
}

// TinyMatrix3x3::getRotation, src/math/tiny/tiny_matrix3x3.h:434-466 (used for the visual outputs)
__device__ void matrix_to_quat_dev(const float* m, float* q) {
  float trace = m[0] + m[4] + m[8];
  float temp[4];
  if (trace < 0.f) {
    int i = m[0] < m[4] ? (m[4] < m[8] ? 2 : 1) : (m[0] < m[8] ? 2 : 0);
    int j = (i + 1) % 3, k = (i + 2) % 3;
    float tmp = ((m[i * 3 + i] - m[j * 3 + j]) - m[k * 3 + k]) + 1.f;
    float s = sqrtf(tmp);
    temp[i] = s * 0.5f;
    s = 0.5f / s;
    temp[3] = (m[j * 3 + k] - m[k * 3 + j]) * s;
    temp[j] = (m[i * 3 + j] + m[j * 3 + i]) * s;
    temp[k] = (m[i * 3 + k] + m[k * 3 + i]) * s;
  } else {
    float s = sqrtf(trace + 1.f);
    temp[3] = s * 0.5f;
    s = 0.5f / s;
    temp[0] = (m[5] - m[7]) * s;
    temp[1] = (m[6] - m[2]) * s;
    temp[2] = (m[1] - m[3]) * s;
  }
  q[0] = temp[0]; q[1] = temp[1]; q[2] = temp[2]; q[3] = -temp[3];
}

// Output packing of LocomotionContactSimulation::step_forward_original,
// examples/environments/locomotion_contact_simulation.h:273-303: q | qd | visuals (pos3, quat4) | up.z
__global__ void pack_v1_output_kernel(const __grid_constant__ DevVisuals V, const float* __restrict__ q,
                                      const float* __restrict__ qd, const float* __restrict__ link_xf,
                                      double* __restrict__ out, int out_dim, int n, int ns, int floating) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  double* o = out + (size_t)e * out_dim;
  int j = 0;
  for (int k = 0; k < V.n_q; ++k) o[j++] = (double)q[(size_t)k * ns + e];
  for (int k = 0; k < V.n_qd; ++k) o[j++] = (double)qd[(size_t)k * ns + e];
  for (int v = 0; v < V.n_vis; ++v) {
    const float* x = link_xf + (size_t)V.v_link[v] * 12 * ns + e;
    float R[9], t[3], Rv[9], q4[4];
    for (int k = 0; k < 9; ++k) R[k] = x[(size_t)k * ns];
    for (int k = 0; k < 3; ++k) t[k] = x[(size_t)(9 + k) * ns];
    for (int r = 0; r < 3; ++r) {
      o[j++] = (double)(t[r] + R[r * 3] * V.v_t[v][0] + R[r * 3 + 1] * V.v_t[v][1] + R[r * 3 + 2] * V.v_t[v][2]);
      for (int c = 0; c < 3; ++c)
        Rv[r * 3 + c] = R[r * 3] * V.v_R[v][c] + R[r * 3 + 1] * V.v_R[v][3 + c] + R[r * 3 + 2] * V.v_R[v][6 + c];
    }
    matrix_to_quat_dev(Rv, q4);
    o[j++] = q4[0]; o[j++] = q4[1]; o[j++] = q4[2]; o[j++] = q4[3];
  }
  double upz = 1.0;  // base_X_world.rotation(2,2): identity for fixed base (:131), else from the new base quat
  if (floating) {
    const double x = q[e], y = q[(size_t)ns + e], z = q[(size_t)2 * ns + e], w = q[(size_t)3 * ns + e];
    upz = 1.0 - 2.0 * (x * x + y * y) / (x * x + y * y + z * z + w * w);
  }
  o[j++] = upz;
}

// Visual-transform stream in the instancing renderer's layout (SURVEY 8f.2): instance i = env * n_vis + v;
// positions[4 i + {0,1,2,3}] = x, y, z, 1 and orientations[4 i + {0..3}] = quaternion xyzw, the two arrays
// TinyGLInstancingRenderer keeps (src/visualizer/opengl/tiny_gl_instancing_renderer.cpp:366-367, 440-457).  Same
// per-visual transform as the v1 output records (locomotion_contact_simulation.h:281-299).
__global__ void pack_visual_instances_kernel(const __grid_constant__ DevVisuals V, const float* __restrict__ link_xf,
                                             float4* __restrict__ positions, float4* __restrict__ orientations, int n, int ns) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  const int v = blockIdx.y;
  if (e >= n) return;
  const float* x = link_xf + (size_t)V.v_link[v] * 12 * ns + e;
  float R[9], t[3], Rv[9], q4[4], p[3];
  for (int k = 0; k < 9; ++k) R[k] = x[(size_t)k * ns];
  for (int k = 0; k < 3; ++k) t[k] = x[(size_t)(9 + k) * ns];
  for (int r = 0; r < 3; ++r) {
    p[r] = t[r] + R[r * 3] * V.v_t[v][0] + R[r * 3 + 1] * V.v_t[v][1] + R[r * 3 + 2] * V.v_t[v][2];
    for (int c = 0; c < 3; ++c)
      Rv[r * 3 + c] = R[r * 3] * V.v_R[v][c] + R[r * 3 + 1] * V.v_R[v][3 + c] + R[r * 3 + 2] * V.v_R[v][6 + c];
  }
  matrix_to_quat_dev(Rv, q4);
  const size_t i = (size_t)e * V.n_vis + v;
  positions[i] = make_float4(p[0], p[1], p[2], 1.f);
  orientations[i] = make_float4(q4[0], q4[1], q4[2], q4[3]);
}

// ---- environment layer on the device (SURVEY 8f.1) ---------------------------------------------------------------
// counter-based uniform in [0, 1): splitmix64 of (seed, environment, joint)
__device__ inline float unit_uniform(unsigned long long seed, unsigned e, unsigned a) {
  unsigned long long z = seed + 0x9E3779B97F4A7C15ull * (((unsigned long long)e << 8) + a + 1ull);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z ^= z >> 31;
  return (float)(z >> 40) * (1.0f / 16777216.0f);
}
// LaikagoContactSimulation::reset, laikago_environment2.h:63-89: reset pose, joint noise on the actuated joints, qd = 0
__global__ void env_reset_fill_kernel(float* __restrict__ q, float* __restrict__ qd, const float* __restrict__ noise, float amp,
                                      unsigned long long seed, EnvParams E, int n_q, int n_qd, const int* __restrict__ act_qidx,
                                      int n, int ns) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  for (int k = 0; k < n_q; ++k) q[(size_t)k * ns + e] = E.reset_q[k];
  for (int k = 0; k < n_qd; ++k) qd[(size_t)k * ns + e] = 0.f;
  for (int a = 0; a < E.n_act; ++a) {
    const float d = noise ? noise[(size_t)a * ns + e] : amp * (2.f * unit_uniform(seed, (unsigned)e, (unsigned)a) - 1.f);
    q[(size_t)act_qidx[a] * ns + e] += d;
  }
}
__global__ void env_select_kernel(const float* __restrict__ mask, const float* __restrict__ q_src, const float* __restrict__ qd_src,
                                  float* __restrict__ q, float* __restrict__ qd, int n_q, int n_qd, int n, int ns) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n || (mask && mask[e] == 0.f)) return;
  for (int k = 0; k < n_q; ++k) q[(size_t)k * ns + e] = q_src[(size_t)k * ns + e];
  for (int k = 0; k < n_qd; ++k) qd[(size_t)k * ns + e] = qd_src[(size_t)k * ns + e];
}
// VectorizedEnvironment::policy (ars_vectorized_environment.h:293-300): one linear layer with bias per environment
// (neural_network.hpp:223-265, parameters = weights [n_act][n_obs] row-major | biases [n_act]); the observation is
// q | qd with x and y zeroed (ars_vectorized_environment.h:285-287).  params: [n_params][ns] on the device.
// One thread per (environment, action): blockIdx.y = action; consecutive threads = consecutive environments, so every
// parameter / state row is read coalesced.
__global__ void policy_linear_kernel(const float* __restrict__ q, const float* __restrict__ qd, const float* __restrict__ params,
                                     float* __restrict__ act, int n_q, int n_qd, int n_act, int n, int ns) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  const int a = blockIdx.y;
  if (e >= n) return;
  const int n_obs = n_q + n_qd;
  float s = params[(size_t)(n_act * n_obs + a) * ns + e];
  const float* w = params + (size_t)a * n_obs * ns + e;
#pragma unroll 4
  for (int k = 2; k < n_q; ++k) s += q[(size_t)k * ns + e] * w[(size_t)k * ns];
#pragma unroll 4
  for (int k = 0; k < n_qd; ++k) s += qd[(size_t)k * ns + e] * w[(size_t)(n_q + k) * ns];
  act[(size_t)a * ns + e] = s;
}
// ARSVectorizedWorker::rollouts bookkeeping (ars_vectorized_worker.h:117-139): done is sticky, rewards and step counts
// accumulate only while the environment is alive
__global__ void rollout_accum_kernel(const float* __restrict__ reward, const float* __restrict__ done, float shift,
                                     float* __restrict__ sticky, float* __restrict__ total, int* __restrict__ steps, int n) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  if (sticky[e] != 0.f) return;
  if (done[e] != 0.f) { sticky[e] = 1.f; return; }
  total[e] += reward[e] - shift;
  steps[e] += 1;
}
// Contact-pair index list of one step, in the reference's enumeration order (World::compute_contacts_multi_body_internal,
// src/world.hpp:212-281: bodies i < j, links of A, geoms of A, links of B, geoms of B, points in emission order).  The
// candidate points of a model are static (every sphere / capsule end emits one point, contact_point.hpp:112-124,149-158);
// what varies per environment is which of them the constraint solver keeps: all with keep_all_points_, else those with
// distance < 0 (MultiBodyConstraintSolver::resolve_collision, src/mb_constraint_solver.hpp:169-180).
// links: [2 * n_points][ns] = (link_a, link_b) of the k-th kept point (MultiBodyContactPoint::link_a/b, :29-40), -9 beyond count.
// cand (optional): [n_points][ns] index of the k-th kept point in the candidate list (tds_b200_contact_pairs), -9 beyond count.
// A distance of +inf marks a candidate between multibodies whose contact function emitted nothing (contact_point.hpp:80).
__global__ void contact_list_kernel(const float* __restrict__ dist, ContactCandTable T, int keep_all, int* __restrict__ count,
                                    int* __restrict__ links, int* __restrict__ cand, int n, int ns) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  int k = 0;
  for (int c = 0; c < T.n_points; ++c) {
    const float d = dist[(size_t)c * ns + e];
    if (d < 3.0e38f && (keep_all || d < 0.f)) {
      links[(size_t)(2 * k) * ns + e] = T.link_a[c];
      links[(size_t)(2 * k + 1) * ns + e] = T.link_b[c];
      if (cand) cand[(size_t)k * ns + e] = c;
      ++k;
    }
  }
  count[e] = k;
  for (; k < T.n_points; ++k) {
    links[(size_t)(2 * k) * ns + e] = -9; links[(size_t)(2 * k + 1) * ns + e] = -9;
    if (cand) cand[(size_t)k * ns + e] = -9;
  }
}
// integrate_euler (src/dynamics/integrator.hpp:10-133) and integrate_euler_qdd (:141-195) as stand-alone stages of the
// fine-grained pytinydiffsim surface (forward_dynamics -> integrate_euler_qdd -> World::step -> integrate_euler): the fused
// step kernels do the same arithmetic in their epilogues.  qdd may be null (= the zero vector integrate_euler_qdd leaves).
struct IntegrateTable { int n_links, floating, n_q, n_qd; signed char q_idx[TDS_MAX_LINKS], qd_idx[TDS_MAX_LINKS], fixed[TDS_MAX_LINKS]; };
__global__ void integrate_euler_kernel(float* __restrict__ q, float* __restrict__ qd, const float* __restrict__ qdd, double dt,
                                       IntegrateTable T, int update_q, int n, int ns) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  auto Q = [&](int k) -> float& { return q[(size_t)k * ns + e]; };
  auto QD = [&](int k) -> float& { return qd[(size_t)k * ns + e]; };
  if (qdd) for (int k = 0; k < T.n_qd; ++k) QD(k) = (float)((double)QD(k) + (double)qdd[(size_t)k * ns + e] * dt);
  if (!update_q) return;
  if (T.floating) {   // quat_velocity + quat_increment + normalize (tiny_algebra.hpp:604-614)
    const double h = 0.5 * dt;
    double qx = Q(0), qy = Q(1), qz = Q(2), qw = Q(3);
    const double w0 = QD(0), w1 = QD(1), w2 = QD(2);
    const double dw = (-qx * w0 - qy * w1 - qz * w2) * h, dx = (qw * w0 + qz * w1 - qy * w2) * h;
    const double dy = (qw * w1 + qx * w2 - qz * w0) * h, dz = (qw * w2 + qy * w0 - qx * w1) * h;
    qx += dx; qy += dy; qz += dz; qw += dw;
    const double len = sqrt(qx * qx + qy * qy + qz * qz + qw * qw);
    Q(0) = (float)(qx / len); Q(1) = (float)(qy / len); Q(2) = (float)(qz / len); Q(3) = (float)(qw / len);
    for (int k = 0; k < 3; ++k) Q(4 + k) = (float)((double)Q(4 + k) + (double)QD(3 + k) * dt);
  }
  for (int i = 0; i < T.n_links; ++i)
    if (!T.fixed[i]) Q(T.q_idx[i]) = (float)((double)Q(T.q_idx[i]) + (double)QD(T.qd_idx[i]) * dt);
}
// ---- ARS on the device (examples/ars/ars_vectorized_worker.h, ars_learner.h) --------------------------------------
// Observation filter statistics, ars_vectorized_worker.h:93-110: every rollout step pushes the observation the policy saw
// (q | qd with x, y zeroed) into a per-(environment, component) RunningStat (running_stat.h:17-37, Welford).
// stats: [3 * n_obs][ns] = count | mean | S per component; sticky (may be null): finished environments stop pushing -
// the reference keeps pushing the frozen observation of a done environment, which only inflates its count; documented.
__global__ void obs_stat_push_kernel(const float* __restrict__ q, const float* __restrict__ qd, float* __restrict__ stats,
                                     int n_q, int n_qd, int n, int ns) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  const int o = blockIdx.y;
  if (e >= n) return;
  const int n_obs = n_q + n_qd;
  float x = o < n_q ? q[(size_t)o * ns + e] : qd[(size_t)(o - n_q) * ns + e];
  if (o < 2) x = 0.f;                                   // ars_vectorized_environment.h:285-287
  float* cnt = stats + (size_t)o * ns + e;
  float* mean = stats + (size_t)(n_obs + o) * ns + e;
  float* S = stats + (size_t)(2 * n_obs + o) * ns + e;
  const float c = *cnt + 1.f;
  if (c == 1.f) { *mean = x; *S = 0.f; }
  else { const float m0 = *mean, m1 = m0 + (x - m0) / c; *S += (x - m0) * (x - m1); *mean = m1; }
  *cnt = c;
}
// per-environment policy parameters of a perturbed rollout: params[p][e] = w[p] + sign * delta_std * delta[p][e]
// (ARSVectorizedWorker::do_rollouts, ars_vectorized_worker.h:205-262)
__global__ void ars_perturb_kernel(const float* __restrict__ w, const float* __restrict__ deltas, float scale,
                                   float* __restrict__ params, int n, int ns) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  const int p = blockIdx.y;
  if (e >= n) return;
  params[(size_t)p * ns + e] = w[p] + scale * deltas[(size_t)p * ns + e];
}
// ARSLearner::weighted_sum_custom + train_step (ars_learner.h:67-91,185-189): g_hat[p] = (1 / N) sum_e (r+ - r-)[e]
// delta[p][e] delta_std ; w[p] += step_size g_hat[p].  One block per parameter, tree reduction over the environments.
__global__ void ars_update_kernel(float* __restrict__ w, const float* __restrict__ deltas, const float* __restrict__ r_pos,
                                  const float* __restrict__ r_neg, float delta_std, float step_size, int n, int ns) {
  __shared__ float red[256];
  const int p = blockIdx.x;
  float acc = 0.f;
  for (int e = threadIdx.x; e < n; e += blockDim.x) acc += (r_pos[e] - r_neg[e]) * deltas[(size_t)p * ns + e];
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int s = blockDim.x / 2; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) w[p] += step_size * (red[0] * delta_std / (float)n);
}
__global__ void rollout_init_kernel(float* sticky, float* total, int* steps, int n) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e < n) { sticky[e] = 0.f; total[e] = 0.f; steps[e] = 0; }
}

}  // namespace

struct tds_b200_sim {
  int device = 0;
  int n = 0, ns = 0;
  DevModel dm[3];         // one layout per precision mode
  DevModel dm_ad;         // layout of the differentiable instance (dual numbers, 16-byte scalars)
  char* jac_scratch = nullptr; size_t jac_scratch_bytes = 0;
  double* jac_dev = nullptr; size_t jac_dev_bytes = 0;   // host paths' Jacobians, tangents and values; the ID device JVP's tangents
  // vector-Jacobian product: tape capacity in nodes per lane (grows by doubling when a run overflows, and stays grown),
  // its node / adjoint / arena buffers, the overflow flag, device staging of the host path
  int tape_cap = 4096;
  char* vjp_buf = nullptr; size_t vjp_buf_bytes = 0;
  int* vjp_flag = nullptr;
  double* vjp_g = nullptr; size_t vjp_g_bytes = 0;   // (also the cotangents G | g of the dynamics queries' VJPs)
  DevModel dm_m;          // layout of the fp64 mass-matrix instance (8-byte scalars)
  float* wrench_dev = nullptr; size_t wrench_dev_bytes = 0;   // host paths of the step with wrenches: W [6K][ns] fp32
  double* mass_dev = nullptr; size_t mass_dev_bytes = 0; // dynamics queries' VJPs: identity tangents | output columns of a chunk
  double* minv_dev = nullptr; size_t minv_dev_bytes = 0; // the inverse mass matrix's intermediates: M^-1, J and their tangents
  double* cdyn_dev = nullptr; size_t cdyn_dev_bytes = 0; // the constrained dynamics' intermediates: h, M^-1, J, drift, solve, tangents
                                                         // (and those of the forward dynamics' derivatives)
  // installed physical parameters (tds_b200_set_physical_params_*): slot map (par.n == 0: none) and values [k][ns] fp64
  ParMap par;
  double* par_dev = nullptr; size_t par_dev_bytes = 0;
  bool smem_ok[3] = {false, false, false};
  bool smem_ok_w[3] = {false, false, false};
  // 3: role-warp kernel (tds_stepr.cu), 2: lane-team kernel (tds_stept.cu), 1: one-lane world-frame kernel
  // (tds_stepw.cu).  Requests fall back 3 -> 2 -> 1 when the model has no
  // tree decomposition (chains) or a tile does not fit in shared memory.
  // 4: ahead-of-time specialised kernel (tds_steps.cu) when the model is one it was generated for, else 3.
  int kernel = 4;
  int kernel_req = 4;
  bool spec_ok = false;
  int spec_idx = -1;       // which compiled model (tds_steps.cu) equals this simulator's, -1: none
  std::vector<double> model;   // flat model (identity check of the specialised kernel)
  bool smem_ok_r[3] = {false, false, false};
  unsigned long long table_token = 0;
  bool team_ok = false;
  bool smem_ok_t[3] = {false, false, false};
  TeamModel tm[3];
  std::vector<TeamLink> team_table;
  TeamLink* team_dev = nullptr;
  int warps_per_block[3] = {1, 1, 1};
  DevVisuals vis;
  SimParams P;
  EnvParams E;
  int precision_req = TDS_B200_PREC_AUTO;   // what the caller asked for
  int precision = TDS_B200_PREC_F64;        // what runs: AUTO resolves to MIXED for a model with a compiled (validated)
                                            // instance, else to the strict F64 (rebuild_team)
  int n_tau = 0, n_points = 0;
  ContactCandTable cand;              // static candidate table (reference enumeration order)
  int *c_count = nullptr, *c_links = nullptr, *c_cand = nullptr;   // device: per-environment contact list of the last tds_b200_contact_list_* call
  size_t c_count_bytes = 0, c_links_bytes = 0, c_cand_bytes = 0;
  // resident state + staging
  float *q = nullptr, *qd = nullptr, *act = nullptr, *qdd = nullptr, *reward = nullptr, *done = nullptr;
  float *cdist = nullptr, *link_xf = nullptr;
  char* scratch = nullptr;
  size_t scratch_bytes = 0;
  void* stage_dev = nullptr;   // device staging for AoS host buffers
  size_t stage_dev_bytes = 0;
  cudaStream_t stream = nullptr;
  int max_smem_optin = 0;
  long long* phase_clk = nullptr;  // profiling only (tds_b200_debug_phase_clocks)
  long long* phase_clk_dev = nullptr;   // profiling only: caller-owned record that replaces phase_clk (tds_b200_debug_phase_clocks_device)
  // tds_b200_env_step_host with pinned caller buffers: the copy / transpose / step / copy sequence is captured once
  // per buffer set and replayed (one graph launch instead of nine stream operations)
  // environment layer scratch: reset staging, zero actions, actuated coordinate map, rollout bookkeeping
  float *rq = nullptr, *rqd = nullptr, *zero_act = nullptr, *pol_act = nullptr, *sticky = nullptr, *r_total = nullptr, *pol_params = nullptr;
  int *act_qidx = nullptr, *r_steps = nullptr;
  float* obs_stats = nullptr;      // caller-owned [3 * n_obs][ns] running statistics of the observation filter, or null
  bool act_qidx_valid = false;
  size_t pol_params_bytes = 0;
  // set around the step launch of tds_b200_env_step_host when the specialised kernel serves the host layouts itself
  const float* io_act_aos = nullptr; float* io_obs_aos = nullptr; float* io_obs_tail = nullptr;
  const void* zc_key[4] = {nullptr, nullptr, nullptr, nullptr};   // zero-copy path: last buffer set and its device aliases
  void* zc_dev[4] = {nullptr, nullptr, nullptr, nullptr};
  bool zc_ok = false;
  unsigned zc_calls = 0;          // the cached classification is re-validated every 64 calls
  const void* g_key[4] = {nullptr, nullptr, nullptr, nullptr};
  int g_seen = 0;
  cudaGraphExec_t g_exec = nullptr;
};

static void drop_host_graph(tds_b200_sim* s) {
  if (s->g_exec) { cudaGraphExecDestroy(s->g_exec); s->g_exec = nullptr; }
  s->g_seen = 0;
  s->g_key[0] = s->g_key[1] = s->g_key[2] = s->g_key[3] = nullptr;
}

static bool is_pinned(const void* p) {
  if (!p) return true;
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
  return a.type == cudaMemoryTypeHost;
}

static int ensure_stage(tds_b200_sim* s, size_t bytes) {
  if (bytes > s->stage_dev_bytes) {
    // the graph of tds_b200_env_step_host holds addresses inside the staging buffer: it dies with the buffer
    drop_host_graph(s);
    CUDA_TRY(grow_dev(&s->stage_dev, &s->stage_dev_bytes, bytes));
  }
  return 0;
}

static int ensure_scratch(tds_b200_sim* s, int prec) {
  const int words = s->dm[prec].w_total > s->dm[prec].x_total ? s->dm[prec].w_total : s->dm[prec].x_total;
  CUDA_TRY(grow_dev(&s->scratch, &s->scratch_bytes, (size_t)words * 4 * s->ns));
  return 0;
}

// Entry of a host path that reuses the simulator's derivative buffers (jac_scratch, jac_dev, vjp_g, mass_dev): selects the
// device and waits for device work already queued.  A device entry point of this simulator may still be running on a caller's
// stream with these buffers, and the simulator's own stream, which the host path runs on, is not ordered against that stream.
static int enter_derivative_host(tds_b200_sim* s) {
  CUDA_TRY(cudaSetDevice(s->device));
  CUDA_TRY(cudaDeviceSynchronize());
  return 0;
}

// ---- fp32 state of the host paths: fp64 host [n][dim] <-> the resident fp32 [dim][ns] buffers, through stage_dev on the
// simulator's stream

// src [n][dim] -> dst [dim][ns]; stage_dev holds n * dim doubles
static int put_state(tds_b200_sim* s, const double* src, int dim, float* dst) {
  if (dim == 0) return 0;
  CUDA_TRY(cudaMemcpyAsync(s->stage_dev, src, sizeof(double) * s->n * dim, cudaMemcpyHostToDevice, s->stream));
  aos_to_soa_kernel<double><<<(s->n + 127) / 128, 128, 0, s->stream>>>((const double*)s->stage_dev, dim, 0, dst, dim, s->n, s->ns);
  return 0;
}

// q -> s->q, with stage_dev sized for any one state array of the host paths (q, qd, the step's inputs, the contact distances)
static int put_q(tds_b200_sim* s, const double* q) {
  const DevModel& M = s->dm[0];
  const size_t rows = (size_t)(M.n_q > M.n_qd ? M.n_q : M.n_qd) + s->n_points + 1;
  if (int rc = ensure_stage(s, sizeof(double) * s->n * rows)) return rc;
  return put_state(s, q, M.n_q, s->q);
}

// q, qd and the step's inputs (NULL: zero) -> s->q, s->qd, s->act
static int put_step_inputs(tds_b200_sim* s, int use_pd, const double* q, const double* qd, const double* tau_or_action) {
  const int n_in = use_pd ? s->E.n_act : s->n_tau;
  int rc = put_q(s, q);
  if (!rc) rc = put_state(s, qd, s->dm[0].n_qd, s->qd);
  if (rc) return rc;
  if (tau_or_action) return put_state(s, tau_or_action, n_in, s->act);
  CUDA_TRY(cudaMemsetAsync(s->act, 0, sizeof(float) * s->ns * (n_in > 0 ? n_in : 1), s->stream));
  return 0;
}

// src [dim][ns] -> dst [n][dim] (dst NULL: nothing); returns with dst written
static int get_state(tds_b200_sim* s, const float* src, int dim, double* dst) {
  if (dim == 0 || !dst) return 0;
  if (int rc = ensure_stage(s, sizeof(double) * s->n * dim)) return rc;
  soa_to_aos_kernel<double><<<(s->n + 127) / 128, 128, 0, s->stream>>>(src, (double*)s->stage_dev, dim, 0, dim, s->n, s->ns);
  CUDA_TRY(cudaMemcpyAsync(dst, s->stage_dev, sizeof(double) * s->n * dim, cudaMemcpyDeviceToHost, s->stream));
  CUDA_TRY(cudaStreamSynchronize(s->stream));
  return 0;
}

// (Re)build the team decomposition: depends on the model and on the action -> link map of the environment.
static int rebuild_team(tds_b200_sim* s) {
  s->team_ok = false;
  s->spec_ok = false; s->spec_idx = -1;
  TeamModel base;
  if (s->precision_req == TDS_B200_PREC_AUTO) s->precision = TDS_B200_PREC_F64;
  if (s->dm[0].world_only) return 0;   // box shapes / spherical joints: the generic world-frame kernel serves the model
  int rc = tds_build_team(&s->dm[0], &s->E, &base, &s->team_table);
  if (rc != 0) return 0;   // chains etc.: the one-lane kernel is used
  const int sizes[3][3] = {{4, 8, 4}, {8, 8, 8}, {4, 4, 4}};
  for (int p = 0; p < 3; ++p) {
    s->tm[p] = base;
    tds_build_team_layout(&s->tm[p], sizes[p][0], sizes[p][1], sizes[p][2]);
    s->smem_ok_t[p] = tds_stept_tile_bytes(&s->tm[p]) <= (size_t)s->max_smem_optin;
    s->smem_ok_r[p] = tds_stepr_tile_bytes(&s->tm[p]) <= (size_t)s->max_smem_optin;
  }
  static unsigned long long next_token = 1;
  s->table_token = next_token++;
  s->spec_idx = tds_spec_find(s->model.data(), (int)s->model.size(), &s->dm[0], &s->E);
  s->spec_ok = s->spec_idx >= 0;
  if (s->precision_req == TDS_B200_PREC_AUTO) s->precision = s->spec_ok ? TDS_B200_PREC_MIXED : TDS_B200_PREC_F64;
  if (!s->team_dev) CUDA_TRY(cudaMalloc((void**)&s->team_dev, sizeof(TeamLink) * TDS_TEAM_T * TDS_TEAM_MAXK));
  CUDA_TRY(cudaMemcpy(s->team_dev, s->team_table.data(), sizeof(TeamLink) * TDS_TEAM_T * TDS_TEAM_MAXK, cudaMemcpyHostToDevice));
  s->team_ok = true;
  return 0;
}

extern "C" {

static const char* tds_model_error(int rc) {
  switch (rc) {
    case -1: return "not a flat model of this layout version (magic / size mismatch)";
    case -2: return "too many links, collision geoms or candidate contact points (TDS_MAX_LINKS / TDS_MAX_GEOMS / TDS_MAX_POINTS)";
    case -3: return "unknown joint type";
    case -4: return "links are not ordered parent before child";
    case -5: return "collision geoms are not grouped by link";
    case -6: return "mesh collision shape against the ground plane: the contact stage implements sphere, capsule and box";
    case -7: return "world of several multibodies (TDSM_H_NBODIES): fixed base only, links of a multibody contiguous, as many root links as multibodies";
    default: return "unknown error";
  }
}

// Host-only check (no GPU needed): 0 when tds_b200_create would accept the model, else the negative code; the reason
// is left in tds_b200_last_error().
int tds_b200_validate_model(const double* model, int n_model) {
  if (!model) { set_err("null model"); return -1; }
  DevModel* D = new DevModel;
  const int rc = tds_build_dev_model(model, n_model, D);
  delete D;
  if (rc) set_err(std::string("unsupported model: ") + tds_model_error(rc));
  return rc;
}

tds_b200_sim* tds_b200_create(const double* model, int n_model, int n_envs, int device) {
  if (!model || n_envs <= 0) { set_err("bad arguments"); return nullptr; }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    set_err("no CUDA device available: libtds_b200 has no CPU fallback");
    return nullptr;
  }
  if (cudaSetDevice(device) != cudaSuccess) { set_err("cudaSetDevice failed"); return nullptr; }
  tds_b200_sim* s = new tds_b200_sim;
  s->device = device;
  s->n = n_envs;
  s->ns = (n_envs + 31) & ~31;
  DevModel base;
  int rc = tds_build_dev_model(model, n_model, &base);
  if (rc) {
    set_err(std::string("unsupported model: ") + tds_model_error(rc));
    delete s;
    return nullptr;
  }
  cudaDeviceGetAttribute(&s->max_smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
  const int sizes[3][3] = {{4, 8, 4}, {8, 8, 8}, {4, 4, 4}};  // sizeof(RA, RC, RS) per precision mode
  for (int p = 0; p < 3; ++p) {
    s->dm[p] = base;
    tds_build_layout(&s->dm[p], sizes[p][0], sizes[p][1], sizes[p][2], -1);
    tds_build_layout_w(&s->dm[p], sizes[p][0], sizes[p][1], sizes[p][2], -1);
    size_t per_warp = (size_t)s->dm[p].w_total * 32 * 4;
    s->smem_ok[p] = per_warp <= (size_t)s->max_smem_optin;
    s->smem_ok_w[p] = (size_t)s->dm[p].x_total * 32 * 4 <= (size_t)s->max_smem_optin;
    // several warps per block only help when many blocks would otherwise be needed per SM
    s->warps_per_block[p] = 1;
  }
  s->dm_ad = base;
  tds_build_layout_w(&s->dm_ad, 16, 16, 16, -1, 16);
  s->dm_m = base;
  tds_build_layout_w(&s->dm_m, 8, 8, 8, -1, 8);
  s->model.assign(model, model + n_model);
  { const char* e = nullptr; tds_build_par_map(&base, 0, nullptr, &s->par, &e); }
  if (const char* kv = getenv("TDS_B200_KERNEL"))
    s->kernel_req = strcmp(kv, "world") == 0 ? 1 : (strcmp(kv, "team") == 0 ? 2 : (strcmp(kv, "role") == 0 ? 3 : 4));
  s->kernel = s->kernel_req;
  s->n_tau = base.n_qd - (base.floating ? 6 : 0);
  s->n_points = base.max_contacts + base.n_pair_points;
  s->cand = make_cand_table(base);
  // visuals for the v1 output packing
  memset(&s->vis, 0, sizeof(s->vis));
  {
    const double* vis = model + TDSM_HEADER + TDSM_BASE + (size_t)base.n_links * TDSM_LINK + (size_t)base.n_geoms * TDSM_GEOM;
    int nv = base.n_vis < TDS_MAX_VIS ? base.n_vis : TDS_MAX_VIS;
    s->vis.n_vis = nv; s->vis.n_links = base.n_links; s->vis.n_q = base.n_q; s->vis.n_qd = base.n_qd;
    for (int v = 0; v < nv; ++v) {
      const double* r = vis + (size_t)v * TDSM_VIS;
      s->vis.v_link[v] = (int)r[TDSM_V_LINK];
      for (int k = 0; k < 9; ++k) s->vis.v_R[v][k] = (float)r[TDSM_V_R + k];
      for (int k = 0; k < 3; ++k) s->vis.v_t[v][k] = (float)r[TDSM_V_T + k];
    }
  }
  // defaults = the reference's (world.hpp:65-72, mb_constraint_solver.hpp:59-70)
  s->P.dt = 1e-3; s->P.inv_dt = 1.0 / s->P.dt;
  s->P.gravity[0] = 0; s->P.gravity[1] = 0; s->P.gravity[2] = -9.81;
  s->P.friction = 0.5; s->P.restitution = 0.0; s->P.erp = 0.2; s->P.cfm = 1e-5;
  s->P.pgs_iterations = 1; s->P.keep_all_points = 0;
  s->P.contact_model = 0; s->P.hard_contact_condition = 1;
  s->P.spring_k = 50000.0; s->P.damper_d = 5000.0; s->P.exponent_n = 1.5; s->P.v_transition = 0.01;
  memset(&s->E, 0, sizeof(s->E));
  const size_t ns = s->ns;
  auto alloc = [&](float** p, size_t rows) { return cudaMalloc((void**)p, sizeof(float) * rows * ns) == cudaSuccess && cudaMemset(*p, 0, sizeof(float) * rows * ns) == cudaSuccess; };
  bool ok = alloc(&s->q, base.n_q > 0 ? base.n_q : 1) && alloc(&s->qd, base.n_qd > 0 ? base.n_qd : 1) &&
            alloc(&s->act, (base.n_qd > TDS_MAX_ACT ? base.n_qd : TDS_MAX_ACT)) && alloc(&s->qdd, base.n_qd > 0 ? base.n_qd : 1) &&
            alloc(&s->reward, 1) && alloc(&s->done, 1) && alloc(&s->cdist, s->n_points > 0 ? s->n_points : 1) &&
            alloc(&s->link_xf, (size_t)(base.n_links > 0 ? base.n_links : 1) * 12);
  if (!ok || cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking) != cudaSuccess || rebuild_team(s) != 0) {
    set_err("device allocation failed");
    tds_b200_destroy(s);
    return nullptr;
  }
  return s;
}

void tds_b200_destroy(tds_b200_sim* s) {
  if (!s) return;
  cudaSetDevice(s->device);
  cudaFree(s->q); cudaFree(s->qd); cudaFree(s->act); cudaFree(s->qdd); cudaFree(s->reward); cudaFree(s->done);
  drop_host_graph(s);
  cudaFree(s->rq); cudaFree(s->rqd); cudaFree(s->zero_act); cudaFree(s->pol_act); cudaFree(s->sticky); cudaFree(s->r_total);
  cudaFree(s->pol_params); cudaFree(s->act_qidx); cudaFree(s->r_steps);
  cudaFree(s->c_count); cudaFree(s->c_links); cudaFree(s->c_cand); cudaFree(s->jac_scratch); cudaFree(s->jac_dev);
  cudaFree(s->vjp_buf); cudaFree(s->vjp_flag); cudaFree(s->vjp_g); cudaFree(s->par_dev); cudaFree(s->mass_dev); cudaFree(s->minv_dev); cudaFree(s->wrench_dev);
  cudaFree(s->cdyn_dev);
  cudaFree(s->cdist); cudaFree(s->link_xf); cudaFree(s->scratch); cudaFree(s->stage_dev); cudaFree(s->phase_clk); cudaFree(s->team_dev);
  if (s->stream) cudaStreamDestroy(s->stream);
  delete s;
}

int tds_b200_set_params(tds_b200_sim* s, double dt, const double gravity[3], double friction, double restitution,
                        double erp, double cfm, int pgs_iterations, int keep_all_points) {
  if (!s) return -1;
  drop_host_graph(s);
  s->P.dt = dt; s->P.inv_dt = 1.0 / dt;
  for (int k = 0; k < 3; ++k) s->P.gravity[k] = gravity[k];
  s->P.friction = friction; s->P.restitution = restitution; s->P.erp = erp; s->P.cfm = cfm;
  s->P.pgs_iterations = pgs_iterations; s->P.keep_all_points = keep_all_points;
  return 0;
}

int tds_b200_set_contact_model(tds_b200_sim* s, int contact_model, double spring_k, double damper_d, double exponent_n,
                               double v_transition, int hard_contact_condition) {
  if (!s || contact_model < 0 || contact_model > 1) { set_err("contact_model must be 0 (LCP) or 1 (spring-damper)"); return -1; }
  if (contact_model == 1 && !(spring_k >= 0.0 && damper_d >= 0.0 && exponent_n > 0.0 && v_transition > 0.0)) {
    set_err("spring-damper parameters out of range"); return -2;
  }
  drop_host_graph(s);
  s->P.contact_model = contact_model; s->P.hard_contact_condition = hard_contact_condition ? 1 : 0;
  s->P.spring_k = spring_k; s->P.damper_d = damper_d; s->P.exponent_n = exponent_n; s->P.v_transition = v_transition;
  return 0;
}

int tds_b200_set_env(tds_b200_sim* s, int n_act, const double* initial_poses, int start_link, double kp, double kd,
                     double max_force, double action_limit, int reward_kind) {
  if (!s || n_act < 0 || n_act > TDS_MAX_ACT) { set_err("bad n_act"); return -1; }
  drop_host_graph(s);
  const DevModel& M = s->dm[0];
  EnvParams E;
  memset(&E, 0, sizeof(E));
  E.n_act = n_act; E.start_link = start_link;
  E.kp = (float)kp; E.kd = (float)kd; E.max_force = (float)max_force; E.action_limit = (float)action_limit;
  E.reward_kind = reward_kind;
  int k = 0;
  const int first = M.floating ? 0 : start_link;  // locomotion_contact_simulation.h:181
  for (int i = first; i < M.n_links && k < n_act; ++i) {
    if (M.flags[i] & TDS_LF_FIXED) continue;
    E.act_link[k] = i;
    E.initial_poses[k] = (float)initial_poses[k];
    ++k;
  }
  if (k != n_act) { set_err("model has fewer actuated links than n_act"); return -2; }
  E.auto_reset = s->E.auto_reset;
  memcpy(E.reset_q, s->E.reset_q, sizeof(E.reset_q));
  s->E = E;
  s->act_qidx_valid = false;
  return rebuild_team(s);
}

int tds_b200_set_auto_reset(tds_b200_sim* s, int enable, const double* reset_q) {
  if (!s) return -1;
  const DevModel& M = s->dm[0];
  if (enable && !reset_q) { set_err("auto-reset needs a reset pose"); return -1; }
  drop_host_graph(s);
  s->E.auto_reset = enable ? 1 : 0;
  if (reset_q)
    for (int k = 0; k < M.n_q; ++k) s->E.reset_q[k] = (float)reset_q[k];
  return 0;
}

int tds_b200_set_precision(tds_b200_sim* s, int precision) {
  if (!s || precision < TDS_B200_PREC_AUTO || precision > 2) return -1;
  drop_host_graph(s);
  s->precision_req = precision;
  s->precision = precision != TDS_B200_PREC_AUTO ? precision : (s->spec_ok ? TDS_B200_PREC_MIXED : TDS_B200_PREC_F64);
  return 0;
}

int tds_b200_param_count(const tds_b200_sim* s) { return s ? tds_param_count(&s->dm[0]) : -1; }

// values: device [k][ns] (copied on `stream`) or host [n][k] (synchronous), fp64
static int set_physical_params(tds_b200_sim* s, int k, const int* ids, const double* values, bool device, void* stream) {
  if (!s) return -1;
  if (k > 0 && !values) { set_err("physical params: null values"); return -1; }
  ParMap pm;
  const char* err = nullptr;
  if (tds_build_par_map(&s->dm[0], k, ids, &pm, &err)) { set_err(std::string("physical params: ") + err); return -2; }
  CUDA_TRY(cudaSetDevice(s->device));
  const bool same_ids = memcmp(&pm, &s->par, sizeof(pm)) == 0;   // (the map keeps no pointers: they are set per launch)
  // a captured host graph holds the parameter buffer and the kernel instance: it stays valid only for new values of the same ids
  if (!same_ids) drop_host_graph(s);
  if (k == 0) {
    s->par = pm;
    return 0;
  }
  const size_t bytes = sizeof(double) * (size_t)k * s->ns;
  if (bytes > s->par_dev_bytes) {
    drop_host_graph(s);
    CUDA_TRY(grow_dev(&s->par_dev, &s->par_dev_bytes, bytes));
    CUDA_TRY(cudaMemset(s->par_dev, 0, bytes));
  }
  if (device) {
    CUDA_TRY(cudaMemcpyAsync(s->par_dev, values, bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  } else {
    // steps run on non-blocking streams, which this copy does not wait for
    CUDA_TRY(cudaDeviceSynchronize());
    CUDA_TRY(put_rows(s->par_dev, values, k, s->n, s->ns, s->stream));
    // a copy from pageable memory may return before its DMA has landed, and the non-blocking streams do not wait for it either
    CUDA_TRY(cudaDeviceSynchronize());
  }
  s->par = pm;
  return 0;
}

int tds_b200_set_physical_params_device(tds_b200_sim* s, int k, const int* ids, const double* values, void* stream) {
  return set_physical_params(s, k, ids, values, true, stream);
}

int tds_b200_set_physical_params_host(tds_b200_sim* s, int k, const int* ids, const double* values) {
  return set_physical_params(s, k, ids, values, false, nullptr);
}

int tds_b200_get_dims(const tds_b200_sim* s, int dims[8]) {
  if (!s) return -1;
  const DevModel& M = s->dm[0];
  dims[0] = s->n; dims[1] = s->ns; dims[2] = M.n_q; dims[3] = M.n_qd; dims[4] = s->n_tau; dims[5] = M.n_links;
  dims[6] = s->n_points; dims[7] = s->E.n_act;
  return 0;
}

int tds_b200_step_device(tds_b200_sim* s, int mode, int use_pd, const float* q_in, const float* qd_in,
                         const float* tau_or_action, float* q_out, float* qd_out, float* qdd_out, float* reward,
                         float* done, float* contact_dist, float* link_xf, void* stream) {
  if (!s) return -1;
  const int p = s->precision;
  StepIO io;
  io.q_in = q_in; io.qd_in = qd_in; io.tau_in = tau_or_action;
  io.q_out = q_out; io.qd_out = qd_out; io.qdd_out = qdd_out;
  io.reward = reward; io.done = done; io.contact_dist = contact_dist; io.link_xf = link_xf;
  io.phase_clk = s->phase_clk_dev ? s->phase_clk_dev : s->phase_clk;
  io.act_aos = s->io_act_aos; io.obs_aos = s->io_obs_aos; io.obs_tail = s->io_obs_tail;
  io.jac = nullptr; io.jac_n_in = 0; io.jac_dir0 = 0;
  io.n = s->n; io.n_stride = s->ns;
  if (use_pd && s->E.n_act == 0) { set_err("use_pd without tds_b200_set_env"); return -3; }
  int kern = s->kernel_req;
  if (s->dm[0].world_only || mode == 3 || s->P.contact_model != 0 || s->par.n > 0) kern = 1;   // (mode 3 = TDS_B200_MODE_WORLD)   // box shapes / spherical joints: served by the generic world-frame kernel only
  if (kern == 4 && !(s->spec_ok && tds_spec_smem_bytes(s->spec_idx, p) <= (size_t)s->max_smem_optin)) kern = 3;
  if (kern == 4) {
    s->kernel = kern;
    static const int solo = getenv("TDS_B200_DEBUG_SOLO") ? 256 : 0;   // profiling aid, see tds_steps.cu
    int rcs = tds_launch_step_spec(s->spec_idx, &s->P, &s->E, &io, mode | solo, use_pd, p, (cudaStream_t)stream);
    if (rcs) set_err(std::string("specialised step launch: ") + cudaGetErrorString((cudaError_t)rcs));
    return rcs;
  }
  if (kern == 3 && !(s->team_ok && s->smem_ok_r[p])) kern = 2;
  if (kern == 2 && !s->team_ok) kern = 1;
  s->kernel = kern;
  if (kern == 3) {
    int rcr = tds_launch_stepr(&s->tm[p], s->team_table.data(), s->table_token, &s->dm[p], &s->P, &s->E, &io, mode, use_pd, p,
                               nullptr, 1, (cudaStream_t)stream);
    if (rcr) set_err(std::string("role-warp step launch: ") + cudaGetErrorString((cudaError_t)rcr));
    return rcr;
  }
  if (kern == 2) {
    const int use_smem_t = s->smem_ok_t[p] ? 1 : 0;
    if (!use_smem_t)   // one tile per warp of 32 / TDS_TEAM_T environments
      CUDA_TRY(grow_dev(&s->scratch, &s->scratch_bytes, tds_stept_tile_bytes(&s->tm[p]) * ((s->n + (32 / TDS_TEAM_T) - 1) / (32 / TDS_TEAM_T))));
    int rct = tds_launch_stept(&s->tm[p], s->team_dev, &s->dm[p], &s->P, &s->E, &io, mode, use_pd, p, s->scratch, use_smem_t,
                               (cudaStream_t)stream);
    if (rct) set_err(std::string("team step launch: ") + cudaGetErrorString((cudaError_t)rct));
    return rct;
  }
  const int use_smem = s->smem_ok_w[p] ? 1 : 0;
  if (!use_smem) { int rc = ensure_scratch(s, p); if (rc) return rc; }
  ParMap pm = s->par;
  pm.values = s->par_dev; pm.grad = nullptr;
  int rc = s->par.n > 0
      ? tds_launch_stepw_par(&s->dm[p], &s->P, &s->E, &io, &pm, mode, use_pd, p, s->scratch, use_smem, s->warps_per_block[p],
                             (cudaStream_t)stream)
      : tds_launch_stepw(&s->dm[p], &s->P, &s->E, &io, mode, use_pd, p, s->scratch, use_smem, s->warps_per_block[p], (cudaStream_t)stream);
  if (rc) set_err(std::string("step launch: ") + cudaGetErrorString((cudaError_t)rc));
  return rc;
}

// ---- differentiable step (SURVEY 8f.4): d(q', qd') / d(q, qd, tau | action, kp, kd, max_force), or d qdd / d(...) in
// forward-dynamics mode, by forward-mode dual numbers through the world-frame step kernel (tds_stepw.cu, tds_dual.cuh).
int tds_b200_jacobian_dims(const tds_b200_sim* s, int mode, int use_pd, int dims[2]) {
  if (!s || !dims) return -1;
  const DevModel& M = s->dm[0];
  dims[0] = mode == TDS_B200_MODE_FD ? M.n_qd : M.n_q + M.n_qd;
  dims[1] = M.n_q + M.n_qd + (use_pd ? s->E.n_act + 3 : s->n_tau);
  return 0;
}

// what a Jacobian-vector product differentiates: the step, one of the dynamics queries of DESIGN.md sections 7.12-7.14, 7.16 and 7.17,
// or the step with its contact records (section 7.15)
enum class Query { step, mass, kin, inv, contacts, centroidal, motion, wrench, regressor, minv, cor, der };

// tangents of a Jacobian-vector product: t_in [cols * m][ns], t_par [k * m][ns] (either may be null).  step: t_in = the step's
// inputs; mass: t_in = the q tangents (the step's arguments are not read); kin: the kinematics of the point table and outputs `kin`
// (t_in = the q tangents, t_par unused); inv: t_in = the q | qd | qdd tangents (qd and qdd in the step's qd and tau_or_action);
// contacts: as step, with the rows q' | qd' | records; centroidal: t_in = the q | qd tangents (qd in the step's qd), outputs `cen`;
// motion: t_in = the q | qd | qdd tangents (qd and qdd as for inv), the point table and outputs `mot`; wrench: as step, with the point
// table, wrenches and wrench tangents `ext`; regressor: t_in = the q | qd | qdd tangents (as for inv), Y in jac and the
// energy outputs `reg`; minv: as mass, M^-1 in jac; cor: t_in = the q | qd tangents (qd in the step's qd), C in jac; der: t_in as for
// inv, d tau / dq in jac and d tau / dqd in der_dqd (either may be NULL), qdd from the fp64 der_qdd [n_qd][ns] when not NULL
struct JvpTangents {
  const double* t_in; const double* t_par; int m; Query query = Query::step; const TdsKinCall* kin = nullptr;
  const TdsCenCall* cen = nullptr; const TdsMotCall* mot = nullptr; const TdsExtCall* ext = nullptr;
  const TdsRegCall* reg = nullptr; double* der_dqd = nullptr; const double* der_qdd = nullptr;
};

// the installed physical parameters as a launch argument in *pmv, or NULL without any
static const ParMap* installed_par(const tds_b200_sim* s, ParMap* pmv) {
  *pmv = s->par;
  pmv->values = s->par_dev; pmv->grad = nullptr;
  return s->par.n > 0 ? pmv : nullptr;
}

// -4 with "<what> without installed physical parameters" when parameter tangents or cotangents `par` come without any installed
static int par_without_installed(const tds_b200_sim* s, const void* par, const char* what) {
  if (!par || s->par.n > 0) return 0;
  set_err(std::string(what) + " without installed physical parameters");
  return -4;
}

// scratch of one launch of a world-frame instance of layout M over every environment: x_total words per lane
static size_t lane_arena_bytes(const tds_b200_sim* s, const DevModel& M) {
  return (size_t)(s->n + 31) / 32 * (size_t)M.x_total * 32 * 4;
}

// scratch of one launch of the external-wrench instances (tds_wrench.cu) on layout M with RA of size_ra bytes: the grown layout's words
static size_t wrench_arena_bytes(const tds_b200_sim* s, const DevModel& M, int size_ra) {
  int words;
  tds_ext_layout_w(&M, size_ra, &words);
  return (size_t)(s->n + 31) / 32 * (size_t)words * 32 * 4;
}

// scratch of one launch of the dynamics-derivative instances (tds_dynamics_derivatives.cu) on layout M with RC of size_rc bytes
static size_t der_arena_bytes(const tds_b200_sim* s, const DevModel& M, int size_rc) {
  return (size_t)(s->n + 31) / 32 * (size_t)tds_der_layout_w(&M, size_rc) * 32 * 4;
}

// directions (Jacobian columns or tangents) one launch of the dual instance takes: the scratch (arena bytes per direction) stays within
// 2 GB
static int dir_chunk_of(const tds_b200_sim* s, size_t arena) {
  const size_t chunk = ((size_t)2 << 30) / arena;
  return (int)(chunk < 1 ? 1 : (chunk > 65535 ? 65535 : chunk));   // (gridDim.y)
}
static int dir_chunk(const tds_b200_sim* s) { return dir_chunk_of(s, lane_arena_bytes(s, s->dm_ad)); }

// Jacobian columns: the step's inputs (params == false) or the installed physical parameters, which are the dual instance's
// directions dims[1] + s (params == true); or, with jv, the m columns J V of the tangent-seeded instance
static int jacobian_run(tds_b200_sim* s, int mode, int use_pd, const float* q, const float* qd, const float* tau_or_action,
                        double* jac, void* stream, bool params, const JvpTangents* jv = nullptr) {
  int dims[2];
  tds_b200_jacobian_dims(s, mode, use_pd, dims);
  const int n_dirs = jv ? jv->m : (params ? s->par.n : dims[1]), dir_base = (params && !jv) ? dims[1] : 0;
  StepIO io;
  memset(&io, 0, sizeof(io));
  io.q_in = q; io.qd_in = qd; io.tau_in = tau_or_action;
  io.jac = jac; io.jac_n_in = n_dirs;
  io.n = s->n; io.n_stride = s->ns;
  ParMap pmv;
  const ParMap* pm = installed_par(s, &pmv);
  const size_t arena = (jv && jv->query == Query::wrench) ? wrench_arena_bytes(s, s->dm_ad, 16)
                       : (jv && jv->query == Query::der)  ? der_arena_bytes(s, s->dm_ad, 16)
                                                          : lane_arena_bytes(s, s->dm_ad);
  if (jv && jv->query == Query::der) { io.g_in = jv->der_dqd; io.g_out = jv->der_qdd; }
  const int chunk = std::min(dir_chunk_of(s, arena), n_dirs);
  CUDA_TRY(grow_dev(&s->jac_scratch, &s->jac_scratch_bytes, arena * chunk));
  const cudaStream_t sm = (cudaStream_t)stream;
  for (int d0 = 0; d0 < n_dirs; d0 += chunk) {
    io.jac_dir0 = dir_base + d0;
    const int nd = n_dirs - d0 < chunk ? n_dirs - d0 : chunk;
    int rc = 0;
    if (!jv) {
      rc = pm ? tds_launch_stepw_jacobian_par(&s->dm_ad, &s->P, &s->E, &io, pm, mode, use_pd, nd, s->jac_scratch, sm)
              : tds_launch_stepw_jacobian(&s->dm_ad, &s->P, &s->E, &io, mode, use_pd, nd, s->jac_scratch, sm);
    } else {
      switch (jv->query) {
        case Query::step:
          rc = tds_launch_stepw_jvp(&s->dm_ad, &s->P, &s->E, &io, pm, jv->t_in, jv->t_par, jv->m, mode, use_pd, nd, s->jac_scratch, sm);
          break;
        case Query::mass: rc = tds_launch_mass_jvp(&s->dm_ad, &io, pm, jv->t_in, jv->t_par, jv->m, nd, s->jac_scratch, sm); break;
        case Query::kin: rc = tds_launch_kin_jvp(&s->dm_ad, &io, jv->kin, jv->t_in, jv->m, nd, s->jac_scratch, sm); break;
        case Query::inv: rc = tds_launch_inv_jvp(&s->dm_ad, &s->P, &io, pm, jv->t_in, jv->t_par, jv->m, nd, s->jac_scratch, sm); break;
        case Query::contacts:
          rc = tds_launch_contacts_jvp(&s->dm_ad, &s->P, &s->E, &io, pm, jv->t_in, jv->t_par, jv->m, mode, use_pd, nd, s->jac_scratch, sm);
          break;
        case Query::centroidal:
          rc = tds_launch_centroidal_jvp(&s->dm_ad, &io, pm, jv->cen, jv->t_in, jv->t_par, jv->m, nd, s->jac_scratch, sm);
          break;
        case Query::motion: rc = tds_launch_point_motion_jvp(&s->dm_ad, &io, jv->mot, jv->t_in, jv->m, nd, s->jac_scratch, sm); break;
        case Query::wrench:
          rc = tds_launch_wrench_jvp(&s->dm_ad, &s->P, &s->E, &io, pm, jv->ext, jv->t_in, jv->t_par, jv->m, mode, use_pd, nd, s->jac_scratch,
                                     sm);
          break;
        case Query::regressor: rc = tds_launch_regressor_jvp(&s->dm_ad, &s->P, &io, jv->reg, jv->t_in, jv->m, nd, s->jac_scratch, sm); break;
        case Query::minv: rc = tds_launch_mass_inverse_jvp(&s->dm_ad, &io, pm, jv->t_in, jv->t_par, jv->m, nd, s->jac_scratch, sm); break;
        case Query::cor: rc = tds_launch_coriolis_jvp(&s->dm_ad, &io, pm, jv->t_in, jv->t_par, jv->m, nd, s->jac_scratch, sm); break;
        case Query::der:
          rc = tds_launch_dynamics_derivatives_jvp(&s->dm_ad, &s->P, &io, pm, jv->t_in, jv->t_par, jv->m, nd, s->jac_scratch, sm);
          break;
      }
    }
    if (rc) { set_err(std::string(jv ? "jvp launch: " : "jacobian launch: ") + cudaGetErrorString((cudaError_t)rc)); return rc; }
  }
  return 0;
}

// diagnostics of the chunking above: how many directions (Jacobian columns or tangents) one launch takes for this simulator
int tds_b200_jacobian_chunk(const tds_b200_sim* s) { return s ? dir_chunk(s) : -1; }

static int jacobian_check(tds_b200_sim* s, int mode, int use_pd, const void* q, const void* qd, const void* jac, bool params) {
  if (!s || !q || !qd || !jac) return -1;
  if (mode == 3) { set_err("jacobian: modes FD, NOCONTACT, FULL"); return -2; }
  if (use_pd && s->E.n_act == 0) { set_err("use_pd without tds_b200_set_env"); return -3; }
  if (params && s->par.n == 0) { set_err("parameter jacobian: no physical parameters installed"); return -4; }
  return 0;
}

int tds_b200_step_jacobian_device(tds_b200_sim* s, int mode, int use_pd, const float* q, const float* qd, const float* tau_or_action,
                                  double* jac, void* stream) {
  if (int rc = jacobian_check(s, mode, use_pd, q, qd, jac, false)) return rc;
  return jacobian_run(s, mode, use_pd, q, qd, tau_or_action, jac, stream, false);
}

int tds_b200_step_param_jacobian_device(tds_b200_sim* s, int mode, int use_pd, const float* q, const float* qd,
                                        const float* tau_or_action, double* jac, void* stream) {
  if (int rc = jacobian_check(s, mode, use_pd, q, qd, jac, true)) return rc;
  return jacobian_run(s, mode, use_pd, q, qd, tau_or_action, jac, stream, true);
}

static int jacobian_host(tds_b200_sim* s, int mode, int use_pd, const double* q, const double* qd,
                         const double* tau_or_action, double* jac, bool params) {
  if (int rc = jacobian_check(s, mode, use_pd, q, qd, jac, params)) return rc;
  if (int rc = enter_derivative_host(s)) return rc;
  int dims[2];
  tds_b200_jacobian_dims(s, mode, use_pd, dims);
  if (params) dims[1] = s->par.n;
  const size_t rows = (size_t)dims[0] * dims[1];
  CUDA_TRY(grow_dev(&s->jac_dev, &s->jac_dev_bytes, sizeof(double) * rows * s->ns));
  if (int rc = put_step_inputs(s, use_pd, q, qd, tau_or_action)) return rc;
  CUDA_TRY(cudaMemsetAsync(s->jac_dev, 0, sizeof(double) * rows * s->ns, s->stream));
  if (int rc = jacobian_run(s, mode, use_pd, s->q, s->qd, s->act, s->jac_dev, s->stream, params)) return rc;
  CUDA_TRY(get_rows(jac, s->jac_dev, rows, s->n, s->ns, s->stream));
  return 0;
}

int tds_b200_step_jacobian_host(tds_b200_sim* s, int mode, int use_pd, const double* q, const double* qd,
                                const double* tau_or_action, double* jac) {
  return jacobian_host(s, mode, use_pd, q, qd, tau_or_action, jac, false);
}

int tds_b200_step_param_jacobian_host(tds_b200_sim* s, int mode, int use_pd, const double* q, const double* qd,
                                      const double* tau_or_action, double* jac) {
  return jacobian_host(s, mode, use_pd, q, qd, tau_or_action, jac, true);
}

// ---- Jacobian-vector products: t_out = J V for m tangents V by the tangent-seeded dual instance (tds_stepw_jvp.cu), one lane per
// (environment, tangent), the tangents in chunks as the Jacobian's directions
static int jvp_check(tds_b200_sim* s, int mode, int use_pd, const void* q, const void* qd, const void* tau_or_action, int m,
                     const void* t_in, const void* t_par, const void* t_out) {
  if (!s || !q || !qd || !t_out || m < 1 || (!t_in && !t_par) || (use_pd && !tau_or_action)) return -1;
  if (mode == 3) { set_err("jvp: modes FD, NOCONTACT, FULL"); return -2; }
  if (use_pd && s->E.n_act == 0) { set_err("use_pd without tds_b200_set_env"); return -3; }
  return par_without_installed(s, t_par, "jvp: parameter tangents");
}

int tds_b200_step_jvp_device(tds_b200_sim* s, int mode, int use_pd, const float* q, const float* qd, const float* tau_or_action,
                             int m, const double* t_in, const double* t_par, double* t_out, void* stream) {
  if (int rc = jvp_check(s, mode, use_pd, q, qd, tau_or_action, m, t_in, t_par, t_out)) return rc;
  const JvpTangents jv{t_in, t_par, m};
  return jacobian_run(s, mode, use_pd, q, qd, tau_or_action, t_out, stream, false, &jv);
}

// host JVP of the step (query step) or of the step with its contact records (query contacts, rows q' | qd' | records)
static int step_jvp_host(tds_b200_sim* s, int mode, int use_pd, const double* q, const double* qd, const double* tau_or_action, int m,
                         const double* t_in, const double* t_par, double* t_out, Query query) {
  if (int rc = enter_derivative_host(s)) return rc;
  const int n = s->n, ns = s->ns, k = s->par.n;
  int dims[2];
  tds_b200_jacobian_dims(s, mode, use_pd, dims);
  if (query == Query::contacts) dims[0] += 10 * s->n_points;
  // tangents: host [n][dim][m] <-> device [dim * m][ns]; t_in | t_par | t_out
  const size_t ti = (size_t)(t_in ? dims[1] : 0) * m, tp = (size_t)(t_par ? k : 0) * m, to = (size_t)dims[0] * m;
  CUDA_TRY(grow_dev(&s->jac_dev, &s->jac_dev_bytes, sizeof(double) * (ti + tp + to) * ns));
  if (int rc = put_step_inputs(s, use_pd, q, qd, tau_or_action)) return rc;
  double* tout_d = s->jac_dev + (ti + tp) * ns;
  CUDA_TRY(put_parts<double>(s->jac_dev, {{t_in, ti}, {t_par, tp}, {nullptr, to}}, n, ns, s->stream));
  const JvpTangents jv{t_in ? s->jac_dev : nullptr, t_par ? s->jac_dev + ti * ns : nullptr, m, query};
  if (int rc = jacobian_run(s, mode, use_pd, s->q, s->qd, s->act, tout_d, s->stream, false, &jv)) return rc;
  CUDA_TRY(get_rows(t_out, tout_d, to, n, ns, s->stream));
  return 0;
}

int tds_b200_step_jvp_host(tds_b200_sim* s, int mode, int use_pd, const double* q, const double* qd, const double* tau_or_action,
                           int m, const double* t_in, const double* t_par, double* t_out) {
  if (int rc = jvp_check(s, mode, use_pd, q, qd, tau_or_action, m, t_in, t_par, t_out)) return rc;
  return step_jvp_host(s, mode, use_pd, q, qd, tau_or_action, m, t_in, t_par, t_out, Query::step);
}

// ---- dynamics queries (DESIGN.md sections 7.12-7.14): the mass matrix, forward kinematics and inverse dynamics by the MASS, KIN and
// INV instances of the world-frame kernel.  Each query has one value launch (value_run), its JVP through the Jacobian's chunk loop
// (jacobian_run) and its VJP by identity tangents (vjp_by_eye).

extern "C++" {   // (templates)
// Value of a dynamics query, one lane per environment on the 8-byte layout: launch(io, installed parameters or NULL) with the inputs
// q [n_q][ns] and qd, qdd [n_qd][ns] fp32 (NULL: zero) and the output rows `out` in io
template <typename Launch>
static int value_run(tds_b200_sim* s, const char* what, const float* q, const float* qd, const float* qdd, double* out, Launch launch) {
  StepIO io;
  memset(&io, 0, sizeof(io));
  io.q_in = q; io.qd_in = qd; io.tau_in = qdd; io.jac = out; io.jac_n_in = 1;
  io.n = s->n; io.n_stride = s->ns;
  ParMap pmv;
  CUDA_TRY(grow_dev(&s->jac_scratch, &s->jac_scratch_bytes, lane_arena_bytes(s, s->dm_m)));
  const int rc = launch(&io, installed_par(s, &pmv));
  if (rc) set_err(std::string(what) + " launch: " + cudaGetErrorString((cudaError_t)rc));
  return rc;
}

// VJP of a dynamics query with `rows` output rows: g_in [n_in][ns] and g_par [k][ns] = <G, dO> for the cotangent G [rows][ns], along
// the identity tangents of the n_in inputs and, only when g_par is wanted (not NULL), of the k installed parameters.  jvp(nd, t_in,
// t_par, dO) runs the query's JVP of nd directions into dO [rows * nd][ns]; the directions run in chunks whose tangents and dO stay
// within 1 GB (s->mass_dev).  A direction's dual lane and its contraction do not depend on the other directions or the chunking.
template <typename Jvp>
static int vjp_by_eye(tds_b200_sim* s, const char* what, int n_in, size_t rows, const double* G, double* g_in, double* g_par,
                      cudaStream_t sm, Jvp jvp) {
  const int k = g_par ? s->par.n : 0, ns = s->ns, total = n_in + k;
  const size_t per_dir = sizeof(double) * (rows + total) * ns;   // dO + identity tangents of one direction
  const int chunk = std::min(total, std::max(1, (int)(((size_t)1 << 30) / per_dir)));
  CUDA_TRY(grow_dev(&s->mass_dev, &s->mass_dev_bytes, per_dir * chunk));
  for (int d0 = 0; d0 < total; d0 += chunk) {
    const int nd = std::min(chunk, total - d0);
    double* t_in = s->mass_dev;
    double* t_par = k > 0 ? t_in + (size_t)n_in * nd * ns : nullptr;
    double* dO = t_in + (size_t)total * nd * ns;
    int rc = tds_launch_mass_eye(t_in, t_par, n_in, k, d0, nd, ns, sm);
    if (!rc) rc = jvp(nd, t_in, t_par, dO);
    if (!rc) rc = tds_launch_mass_contract(G, dO, (int)rows, nd, d0, n_in, g_in, g_par, s->n, ns, sm);
    if (rc) { set_err(std::string(what) + " vjp: " + cudaGetErrorString((cudaError_t)rc)); return rc; }
  }
  return 0;
}
}  // extern "C++"

// ---- joint-space mass matrix M(q) (DESIGN.md section 7.12): the MASS instances of the world-frame kernel (tds_mass.cu) ------------------
// M [n_qd * n_qd][ns] from q [n_q][ns] fp32
static int mass_run(tds_b200_sim* s, const float* q, double* Mo, cudaStream_t sm) {
  return value_run(s, "mass matrix", q, nullptr, nullptr, Mo, [&](const StepIO* io, const ParMap* pm) {
    return tds_launch_mass(&s->dm_m, io, pm, s->jac_scratch, sm);
  });
}

static int mass_jvp_run(tds_b200_sim* s, const float* q, int m, const double* t_q, const double* t_par, double* Mo, double* t_M,
                        cudaStream_t sm) {
  if (Mo) { if (int rc = mass_run(s, q, Mo, sm)) return rc; }
  const JvpTangents jv{t_q, t_par, m, Query::mass};
  return jacobian_run(s, TDS_B200_MODE_FULL, 0, q, nullptr, nullptr, t_M, sm, false, &jv);
}

static int mass_vjp_run(tds_b200_sim* s, const float* q, const double* G, double* g_q, double* g_par, cudaStream_t sm) {
  const size_t nn = (size_t)s->dm[0].n_qd * s->dm[0].n_qd;
  return vjp_by_eye(s, "mass matrix", s->dm[0].n_q, nn, G, g_q, g_par, sm, [&](int nd, const double* t_q, const double* t_par, double* dM) {
    return mass_jvp_run(s, q, nd, t_q, t_par, nullptr, dM, sm);
  });
}

int tds_b200_mass_matrix_device(tds_b200_sim* s, const float* q, double* M, void* stream) {
  if (!s || !q || !M) return -1;
  return mass_run(s, q, M, (cudaStream_t)stream);
}

int tds_b200_mass_matrix_host(tds_b200_sim* s, const double* q, double* M) {
  if (!s || !q || !M) return -1;
  if (int rc = enter_derivative_host(s)) return rc;
  const size_t nn = (size_t)s->dm[0].n_qd * s->dm[0].n_qd;
  if (int rc = put_q(s, q)) return rc;
  CUDA_TRY(grow_dev(&s->jac_dev, &s->jac_dev_bytes, sizeof(double) * nn * s->ns));
  if (int rc = mass_run(s, s->q, s->jac_dev, s->stream)) return rc;
  CUDA_TRY(get_rows(M, s->jac_dev, nn, s->n, s->ns, s->stream));
  return 0;
}

static int mass_jvp_check(tds_b200_sim* s, const void* q, int m, const void* t_q, const void* t_par, const void* t_M) {
  if (!s || !q || !t_M || m < 1 || (!t_q && !t_par)) return -1;
  return par_without_installed(s, t_par, "mass matrix jvp: parameter tangents");
}

int tds_b200_mass_matrix_jvp_device(tds_b200_sim* s, const float* q, int m, const double* t_q, const double* t_par, double* M,
                                    double* t_M, void* stream) {
  if (int rc = mass_jvp_check(s, q, m, t_q, t_par, t_M)) return rc;
  return mass_jvp_run(s, q, m, t_q, t_par, M, t_M, (cudaStream_t)stream);
}

int tds_b200_mass_matrix_jvp_host(tds_b200_sim* s, const double* q, int m, const double* t_q, const double* t_par, double* M,
                                  double* t_M) {
  if (int rc = mass_jvp_check(s, q, m, t_q, t_par, t_M)) return rc;
  if (int rc = enter_derivative_host(s)) return rc;
  const int n = s->n, ns = s->ns;
  const size_t nn = (size_t)s->dm[0].n_qd * s->dm[0].n_qd;
  // tangents: host [n][dim][m] <-> device [dim * m][ns]; t_q | t_par | t_M | M
  const size_t tq = (size_t)(t_q ? s->dm[0].n_q : 0) * m, tp = (size_t)(t_par ? s->par.n : 0) * m, to = nn * m;
  if (int rc = put_q(s, q)) return rc;
  CUDA_TRY(grow_dev(&s->jac_dev, &s->jac_dev_bytes, sizeof(double) * (tq + tp + to + nn) * ns));
  double* d = s->jac_dev;
  double* to_d = d + (tq + tp) * ns;
  CUDA_TRY(put_parts<double>(d, {{t_q, tq}, {t_par, tp}}, n, ns, s->stream));
  if (int rc = mass_jvp_run(s, s->q, m, t_q ? d : nullptr, t_par ? d + tq * ns : nullptr, M ? to_d + to * ns : nullptr, to_d, s->stream))
    return rc;
  CUDA_TRY(get_parts<double>({{t_M, to}, {M, nn}}, to_d, n, ns, s->stream));
  return 0;
}

static int mass_vjp_check(tds_b200_sim* s, const void* q, const void* G, const void* g_q, const void* g_par) {
  if (!s || !q || !G || (!g_q && !g_par)) return -1;
  return par_without_installed(s, g_par, "mass matrix vjp: parameter cotangents");
}

int tds_b200_mass_matrix_vjp_device(tds_b200_sim* s, const float* q, const double* G, double* g_q, double* g_par, void* stream) {
  if (int rc = mass_vjp_check(s, q, G, g_q, g_par)) return rc;
  return mass_vjp_run(s, q, G, g_q, g_par, (cudaStream_t)stream);
}

int tds_b200_mass_matrix_vjp_host(tds_b200_sim* s, const double* q, const double* G, double* g_q, double* g_par) {
  if (int rc = mass_vjp_check(s, q, G, g_q, g_par)) return rc;
  if (int rc = enter_derivative_host(s)) return rc;
  const int n = s->n, ns = s->ns, n_q = s->dm[0].n_q, k = s->par.n;
  const size_t nn = (size_t)s->dm[0].n_qd * s->dm[0].n_qd;
  if (int rc = put_q(s, q)) return rc;
  // G | g_q | g_par
  CUDA_TRY(grow_dev(&s->vjp_g, &s->vjp_g_bytes, sizeof(double) * (nn + n_q + k + 1) * ns));
  double* g_d = s->vjp_g + nn * ns;
  CUDA_TRY(put_rows(s->vjp_g, G, nn, n, ns, s->stream));
  if (int rc = mass_vjp_run(s, s->q, s->vjp_g, g_q ? g_d : nullptr, g_par ? g_d + (size_t)n_q * ns : nullptr, s->stream)) return rc;
  CUDA_TRY(get_parts<double>({{g_q, (size_t)n_q}, {g_par, (size_t)k}}, g_d, n, ns, s->stream));
  return 0;
}

// ---- forward kinematics and point Jacobians (DESIGN.md section 7.13): the KIN instances of the world-frame kernel (tds_kin.cu) ---------
// rows of the outputs xf | x | J
struct KinRows { size_t xf, x, J; size_t all() const { return xf + x + J; } };
static KinRows kin_rows(const tds_b200_sim* s, int K) {
  return KinRows{(size_t)s->dm[0].n_links * 12, (size_t)3 * K, (size_t)3 * K * s->dm[0].n_qd};
}

static int kin_check(tds_b200_sim* s, const void* q, int K, const int* links, const double* local) {
  if (!s || !q) return -1;
  if (K < 0 || K > TDS_B200_MAX_KIN_POINTS) { set_err("kinematics: K out of [0, TDS_B200_MAX_KIN_POINTS]"); return -1; }
  if (K > 0 && (!links || !local)) return -1;
  for (int k = 0; k < K; ++k)
    if (links[k] < -1 || links[k] >= s->dm[0].n_links) { set_err("kinematics: a link index out of [-1, n_links)"); return -1; }
  return 0;
}

// fp64 outputs from q [n_q][ns] fp32 (installed parameters do not enter)
static int kin_run(tds_b200_sim* s, const float* q, const TdsKinCall* kc, cudaStream_t sm) {
  return value_run(s, "kinematics", q, nullptr, nullptr, nullptr, [&](const StepIO* io, const ParMap*) {
    return tds_launch_kin(&s->dm_m, io, kc, s->jac_scratch, sm);
  });
}

// m tangents t_q [n_q * m][ns] -> the outputs' columns [rows * m][ns], through the Jacobian's chunk loop
static int kin_jvp_run(tds_b200_sim* s, const float* q, const TdsKinCall* kc, int m, const double* t_q, cudaStream_t sm) {
  const JvpTangents jv{t_q, nullptr, m, Query::kin, kc};
  return jacobian_run(s, TDS_B200_MODE_FULL, 0, q, nullptr, nullptr, nullptr, sm, false, &jv);
}

// g_q = <G, d(xf | x | J)>, G [rows][ns] concatenated
static int kin_vjp_run(tds_b200_sim* s, const float* q, int K, const int* links, const double* local, const double* G, double* g_q,
                       cudaStream_t sm) {
  const KinRows R = kin_rows(s, K);
  const size_t ns = s->ns;
  return vjp_by_eye(s, "kinematics", s->dm[0].n_q, R.all(), G, g_q, nullptr, sm, [&](int nd, const double* t_q, const double*, double* dO) {
    const TdsKinCall kc{K, links, local, dO, dO + R.xf * nd * ns, dO + (R.xf + R.x) * nd * ns};
    return kin_jvp_run(s, q, &kc, nd, t_q, sm);
  });
}

int tds_b200_kinematics_device(tds_b200_sim* s, const float* q, int K, const int* links, const double* local, double* xf, double* x,
                               double* J, void* stream) {
  if (int rc = kin_check(s, q, K, links, local)) return rc;
  if (!xf && !x && !J) return -1;
  const TdsKinCall kc{K, links, local, xf, x, J};
  return kin_run(s, q, &kc, (cudaStream_t)stream);
}

int tds_b200_kinematics_host(tds_b200_sim* s, const double* q, int K, const int* links, const double* local, double* xf, double* x,
                             double* J) {
  if (int rc = kin_check(s, q, K, links, local)) return rc;
  if (!xf && !x && !J) return -1;
  if (int rc = enter_derivative_host(s)) return rc;
  const KinRows R = kin_rows(s, K);
  const int n = s->n, ns = s->ns;
  if (int rc = put_q(s, q)) return rc;
  CUDA_TRY(grow_dev(&s->jac_dev, &s->jac_dev_bytes, sizeof(double) * (R.all() + 1) * ns));
  double* d = s->jac_dev;
  const TdsKinCall kc{K, links, local, xf ? d : nullptr, x ? d + R.xf * ns : nullptr, J ? d + (R.xf + R.x) * ns : nullptr};
  if (int rc = kin_run(s, s->q, &kc, s->stream)) return rc;
  CUDA_TRY(get_parts<double>({{xf, R.xf}, {x, R.x}, {J, R.J}}, d, n, ns, s->stream));
  return 0;
}

static int kin_jvp_check(tds_b200_sim* s, const void* q, int K, const int* links, const double* local, int m, const void* t_q,
                         const void* t_xf, const void* t_x, const void* t_J) {
  if (int rc = kin_check(s, q, K, links, local)) return rc;
  if (m < 1 || !t_q || (!t_xf && !t_x && !t_J)) return -1;
  return 0;
}

int tds_b200_kinematics_jvp_device(tds_b200_sim* s, const float* q, int K, const int* links, const double* local, int m,
                                   const double* t_q, double* t_xf, double* t_x, double* t_J, void* stream) {
  if (int rc = kin_jvp_check(s, q, K, links, local, m, t_q, t_xf, t_x, t_J)) return rc;
  const TdsKinCall kc{K, links, local, t_xf, t_x, t_J};
  return kin_jvp_run(s, q, &kc, m, t_q, (cudaStream_t)stream);
}

int tds_b200_kinematics_jvp_host(tds_b200_sim* s, const double* q, int K, const int* links, const double* local, int m,
                                 const double* t_q, double* t_xf, double* t_x, double* t_J) {
  if (int rc = kin_jvp_check(s, q, K, links, local, m, t_q, t_xf, t_x, t_J)) return rc;
  if (int rc = enter_derivative_host(s)) return rc;
  const int n = s->n, ns = s->ns;
  const KinRows R = kin_rows(s, K);
  // tangents: host [n][rows][m] <-> device [rows * m][ns]; t_q | t_xf | t_x | t_J
  const size_t tq = (size_t)s->dm[0].n_q * m;
  if (int rc = put_q(s, q)) return rc;
  CUDA_TRY(grow_dev(&s->jac_dev, &s->jac_dev_bytes, sizeof(double) * (tq + R.all() * m + 1) * ns));
  double* to_d = s->jac_dev + tq * ns;
  CUDA_TRY(put_rows(s->jac_dev, t_q, tq, n, ns, s->stream));
  const TdsKinCall kc{K, links, local, t_xf ? to_d : nullptr, t_x ? to_d + R.xf * m * ns : nullptr,
                      t_J ? to_d + (R.xf + R.x) * m * ns : nullptr};
  if (int rc = kin_jvp_run(s, s->q, &kc, m, s->jac_dev, s->stream)) return rc;
  CUDA_TRY(get_parts<double>({{t_xf, R.xf * m}, {t_x, R.x * m}, {t_J, R.J * m}}, to_d, n, ns, s->stream));
  return 0;
}

static int kin_vjp_check(tds_b200_sim* s, const void* q, int K, const int* links, const double* local, const void* G_xf, const void* G_x,
                         const void* G_J, const void* g_q) {
  if (int rc = kin_check(s, q, K, links, local)) return rc;
  if (!g_q || (!G_xf && !G_x && !G_J)) return -1;
  return 0;
}

int tds_b200_kinematics_vjp_device(tds_b200_sim* s, const float* q, int K, const int* links, const double* local, const double* G_xf,
                                   const double* G_x, const double* G_J, double* g_q, void* stream) {
  if (int rc = kin_vjp_check(s, q, K, links, local, G_xf, G_x, G_J, g_q)) return rc;
  const cudaStream_t sm = (cudaStream_t)stream;
  const KinRows R = kin_rows(s, K);
  // the concatenated cotangent xf | x | J, zero where a part is NULL
  CUDA_TRY(grow_dev(&s->vjp_g, &s->vjp_g_bytes, sizeof(double) * R.all() * s->ns));
  CUDA_TRY(put_parts_d2d<double>(s->vjp_g, {{G_xf, R.xf}, {G_x, R.x}, {G_J, R.J}}, s->ns, sm));
  return kin_vjp_run(s, q, K, links, local, s->vjp_g, g_q, sm);
}

int tds_b200_kinematics_vjp_host(tds_b200_sim* s, const double* q, int K, const int* links, const double* local, const double* G_xf,
                                 const double* G_x, const double* G_J, double* g_q) {
  if (int rc = kin_vjp_check(s, q, K, links, local, G_xf, G_x, G_J, g_q)) return rc;
  if (int rc = enter_derivative_host(s)) return rc;
  const int n = s->n, ns = s->ns, n_q = s->dm[0].n_q;
  const KinRows R = kin_rows(s, K);
  if (int rc = put_q(s, q)) return rc;
  // G (xf | x | J, zero where a part is NULL) | g_q
  CUDA_TRY(grow_dev(&s->vjp_g, &s->vjp_g_bytes, sizeof(double) * (R.all() + n_q) * ns));
  double* g_d = s->vjp_g + R.all() * ns;
  CUDA_TRY(put_parts<double>(s->vjp_g, {{G_xf, R.xf}, {G_x, R.x}, {G_J, R.J}}, n, ns, s->stream));
  if (int rc = kin_vjp_run(s, s->q, K, links, local, s->vjp_g, g_d, s->stream)) return rc;
  CUDA_TRY(get_rows(g_q, g_d, n_q, n, ns, s->stream));
  return 0;
}

// ---- inverse dynamics tau = ID(q, qd, qdd) (DESIGN.md section 7.14): the INV instances of the world-frame kernel (tds_invdyn.cu) -------
// tau [n_qd][ns] from q [n_q][ns], qd and qdd [n_qd][ns] fp32 (either NULL: zero)
static int inv_run(tds_b200_sim* s, const float* q, const float* qd, const float* qdd, double* tau, cudaStream_t sm) {
  return value_run(s, "inverse dynamics", q, qd, qdd, tau, [&](const StepIO* io, const ParMap* pm) {
    return tds_launch_inv(&s->dm_m, &s->P, io, pm, s->jac_scratch, sm);
  });
}

// inputs of the inverse dynamics' derivatives: q | qd | qdd
static int inv_n_in(const tds_b200_sim* s) { return s->dm[0].n_q + 2 * s->dm[0].n_qd; }

// t_tau [n_qd * m][ns] along t_in [(n_q + 2 n_qd) * m][ns] (q | qd | qdd tangents, contiguous) and t_par (either may be NULL); tau, if
// not NULL, receives the value
static int inv_jvp_run(tds_b200_sim* s, const float* q, const float* qd, const float* qdd, int m, const double* t_in, const double* t_par,
                       double* tau, double* t_tau, cudaStream_t sm) {
  if (tau) { if (int rc = inv_run(s, q, qd, qdd, tau, sm)) return rc; }
  const JvpTangents jv{t_in, t_par, m, Query::inv};
  return jacobian_run(s, TDS_B200_MODE_FULL, 0, q, qd, qdd, t_tau, sm, false, &jv);
}

// g_in [(n_q + 2 n_qd)][ns] (q | qd | qdd, contiguous) and g_par [k][ns] (NULL: not wanted) = G . dtau
static int inv_vjp_run(tds_b200_sim* s, const float* q, const float* qd, const float* qdd, const double* G, double* g_in, double* g_par,
                       cudaStream_t sm) {
  return vjp_by_eye(s, "inverse dynamics", inv_n_in(s), s->dm[0].n_qd, G, g_in, g_par, sm,
                    [&](int nd, const double* t_in, const double* t_par, double* dtau) {
                      return inv_jvp_run(s, q, qd, qdd, nd, t_in, t_par, nullptr, dtau, sm);
                    });
}

// host q [n][n_q], qd and qdd [n][n_qd] (either NULL: zero) -> s->q, s->qd, s->act; the device pointers of qd and qdd (NULL for NULL)
static int put_inv_inputs(tds_b200_sim* s, const double* q, const double* qd, const double* qdd, const float** qd_d, const float** qdd_d) {
  const int nd = s->dm[0].n_qd;
  int rc = put_q(s, q);
  if (!rc && qd) rc = put_state(s, qd, nd, s->qd);
  if (!rc && qdd) rc = put_state(s, qdd, nd, s->act);
  *qd_d = qd ? s->qd : nullptr;
  *qdd_d = qdd ? s->act : nullptr;
  return rc;
}

int tds_b200_inverse_dynamics_device(tds_b200_sim* s, const float* q, const float* qd, const float* qdd, double* tau, void* stream) {
  if (!s || !q || !tau) return -1;
  return inv_run(s, q, qd, qdd, tau, (cudaStream_t)stream);
}

int tds_b200_inverse_dynamics_host(tds_b200_sim* s, const double* q, const double* qd, const double* qdd, double* tau) {
  if (!s || !q || !tau) return -1;
  if (int rc = enter_derivative_host(s)) return rc;
  const int nd = s->dm[0].n_qd;
  const float *qd_d, *qdd_d;
  if (int rc = put_inv_inputs(s, q, qd, qdd, &qd_d, &qdd_d)) return rc;
  CUDA_TRY(grow_dev(&s->jac_dev, &s->jac_dev_bytes, sizeof(double) * (nd + 1) * s->ns));
  if (int rc = inv_run(s, s->q, qd_d, qdd_d, s->jac_dev, s->stream)) return rc;
  CUDA_TRY(get_rows(tau, s->jac_dev, nd, s->n, s->ns, s->stream));
  return 0;
}

static int inv_jvp_check(tds_b200_sim* s, const void* q, int m, const void* t_q, const void* t_qd, const void* t_qdd, const void* t_par,
                         const void* t_tau) {
  if (!s || !q || !t_tau || m < 1 || (!t_q && !t_qd && !t_qdd && !t_par)) return -1;
  return par_without_installed(s, t_par, "inverse dynamics jvp: parameter tangents");
}

int tds_b200_inverse_dynamics_jvp_device(tds_b200_sim* s, const float* q, const float* qd, const float* qdd, int m, const double* t_q,
                                         const double* t_qd, const double* t_qdd, const double* t_par, double* tau, double* t_tau,
                                         void* stream) {
  if (int rc = inv_jvp_check(s, q, m, t_q, t_qd, t_qdd, t_par, t_tau)) return rc;
  const size_t n_q = s->dm[0].n_q, nd = s->dm[0].n_qd;
  cudaStream_t sm = (cudaStream_t)stream;
  double* tin = nullptr;
  if (t_q || t_qd || t_qdd) {   // the kernel reads the q | qd | qdd tangents as one array
    CUDA_TRY(grow_dev(&s->jac_dev, &s->jac_dev_bytes, sizeof(double) * (size_t)inv_n_in(s) * m * s->ns));
    tin = s->jac_dev;
    CUDA_TRY(put_parts_d2d<double>(tin, {{t_q, n_q * m}, {t_qd, nd * m}, {t_qdd, nd * m}}, s->ns, sm));
  }
  return inv_jvp_run(s, q, qd, qdd, m, tin, t_par, tau, t_tau, sm);
}

int tds_b200_inverse_dynamics_jvp_host(tds_b200_sim* s, const double* q, const double* qd, const double* qdd, int m, const double* t_q,
                                       const double* t_qd, const double* t_qdd, const double* t_par, double* tau, double* t_tau) {
  if (int rc = inv_jvp_check(s, q, m, t_q, t_qd, t_qdd, t_par, t_tau)) return rc;
  if (int rc = enter_derivative_host(s)) return rc;
  const int n = s->n, ns = s->ns;
  const size_t n_q = s->dm[0].n_q, nd = s->dm[0].n_qd;
  // tangents: host [n][dim][m] <-> device [dim * m][ns]; q | qd | qdd (contiguous, zero where NULL, none if all are), t_par, dtau, tau
  const size_t ti = (t_q || t_qd || t_qdd) ? (size_t)inv_n_in(s) * m : 0, tp = (size_t)(t_par ? s->par.n : 0) * m, to = nd * m;
  const float *qd_d, *qdd_d;
  if (int rc = put_inv_inputs(s, q, qd, qdd, &qd_d, &qdd_d)) return rc;
  CUDA_TRY(grow_dev(&s->jac_dev, &s->jac_dev_bytes, sizeof(double) * (ti + tp + to + nd + 1) * ns));
  double* d = s->jac_dev;
  double* to_d = d + (ti + tp) * ns;
  if (ti) CUDA_TRY(put_parts<double>(d, {{t_q, n_q * m}, {t_qd, nd * m}, {t_qdd, nd * m}}, n, ns, s->stream));
  if (t_par) CUDA_TRY(put_rows(d + ti * ns, t_par, tp, n, ns, s->stream));
  if (int rc = inv_jvp_run(s, s->q, qd_d, qdd_d, m, ti ? d : nullptr, t_par ? d + ti * ns : nullptr, tau ? to_d + to * ns : nullptr, to_d,
                           s->stream))
    return rc;
  CUDA_TRY(get_parts<double>({{t_tau, to}, {tau, nd}}, to_d, n, ns, s->stream));
  return 0;
}

static int inv_vjp_check(tds_b200_sim* s, const void* q, const void* G, const void* g_q, const void* g_qd, const void* g_qdd,
                         const void* g_par) {
  if (!s || !q || !G || (!g_q && !g_qd && !g_qdd && !g_par)) return -1;
  return par_without_installed(s, g_par, "inverse dynamics vjp: parameter cotangents");
}

int tds_b200_inverse_dynamics_vjp_device(tds_b200_sim* s, const float* q, const float* qd, const float* qdd, const double* G, double* g_q,
                                         double* g_qd, double* g_qdd, double* g_par, void* stream) {
  if (int rc = inv_vjp_check(s, q, G, g_q, g_qd, g_qdd, g_par)) return rc;
  const size_t n_q = s->dm[0].n_q, nd = s->dm[0].n_qd;
  cudaStream_t sm = (cudaStream_t)stream;
  // g_q | g_qd | g_qdd are one array for the contraction: computed in s->vjp_g, then copied out
  CUDA_TRY(grow_dev(&s->vjp_g, &s->vjp_g_bytes, sizeof(double) * (size_t)inv_n_in(s) * s->ns));
  if (int rc = inv_vjp_run(s, q, qd, qdd, G, s->vjp_g, g_par, sm)) return rc;
  CUDA_TRY(get_parts_d2d<double>({{g_q, n_q}, {g_qd, nd}, {g_qdd, nd}}, s->vjp_g, s->ns, sm));
  return 0;
}

int tds_b200_inverse_dynamics_vjp_host(tds_b200_sim* s, const double* q, const double* qd, const double* qdd, const double* G, double* g_q,
                                       double* g_qd, double* g_qdd, double* g_par) {
  if (int rc = inv_vjp_check(s, q, G, g_q, g_qd, g_qdd, g_par)) return rc;
  if (int rc = enter_derivative_host(s)) return rc;
  const int n = s->n, ns = s->ns, n_in = inv_n_in(s);
  const size_t n_q = s->dm[0].n_q, nd = s->dm[0].n_qd, k = s->par.n;
  const float *qd_d, *qdd_d;
  if (int rc = put_inv_inputs(s, q, qd, qdd, &qd_d, &qdd_d)) return rc;
  // G | g_q | g_qd | g_qdd | g_par
  CUDA_TRY(grow_dev(&s->vjp_g, &s->vjp_g_bytes, sizeof(double) * (nd + n_in + k + 1) * ns));
  double* g_d = s->vjp_g + nd * ns;
  CUDA_TRY(put_rows(s->vjp_g, G, nd, n, ns, s->stream));
  if (int rc = inv_vjp_run(s, s->q, qd_d, qdd_d, s->vjp_g, g_d, g_par ? g_d + (size_t)n_in * ns : nullptr, s->stream)) return rc;
  CUDA_TRY(get_parts<double>({{g_q, n_q}, {g_qd, nd}, {g_qdd, nd}, {g_par, k}}, g_d, n, ns, s->stream));
  return 0;
}

// ---- centre of mass, centroidal momentum matrix and its bias (DESIGN.md section 7.16): the CEN instances of the world-frame kernel
// (tds_centroidal.cu) -------------------------------------------------------------------------------------------------------------------
// rows of the outputs com | A | bias
struct CenRows { size_t com, A, bias; size_t all() const { return com + A + bias; } };
static CenRows cen_rows(const tds_b200_sim* s) { return CenRows{10, (size_t)6 * s->dm[0].n_qd, 6}; }

// -2 for the models the query refuses: a world of several multibodies, counted bodies (links, a floating base) without mass
static int cen_model_check(tds_b200_sim* s) {
  const DevModel& M = s->dm[0];
  if (M.n_bodies > 1) { set_err("centroidal: a world of several multibodies (TDSM_H_NBODIES > 1)"); return -2; }
  double m = M.floating ? M.base_rbic[0] : 0.0;
  for (int i = 0; i < M.n_links; ++i) m += M.rbic[i][0];
  if (!(m > 0.0)) { set_err("centroidal: the counted bodies have zero total mass"); return -2; }
  return 0;
}

// fp64 outputs from q [n_q][ns] and qd [n_qd][ns] fp32 (NULL: zero)
static int cen_run(tds_b200_sim* s, const float* q, const float* qd, const TdsCenCall* out, cudaStream_t sm) {
  return value_run(s, "centroidal", q, qd, nullptr, nullptr, [&](const StepIO* io, const ParMap* pm) {
    return tds_launch_centroidal(&s->dm_m, io, pm, out, s->jac_scratch, sm);
  });
}

// inputs of the centroidal derivatives: q | qd
static int cen_n_in(const tds_b200_sim* s) { return s->dm[0].n_q + s->dm[0].n_qd; }

// the outputs' columns [rows * m][ns] along t_in [(n_q + n_qd) * m][ns] (q | qd tangents, contiguous) and t_par (either may be NULL)
static int cen_jvp_run(tds_b200_sim* s, const float* q, const float* qd, int m, const double* t_in, const double* t_par,
                       const TdsCenCall* out, cudaStream_t sm) {
  JvpTangents jv{t_in, t_par, m, Query::centroidal};
  jv.cen = out;
  return jacobian_run(s, TDS_B200_MODE_FULL, 0, q, qd, nullptr, nullptr, sm, false, &jv);
}

// g_in [n_q + n_qd][ns] (q | qd, contiguous) and g_par [k][ns] (NULL: not wanted) = <G, d(com | A | bias)>, G [rows][ns] concatenated
static int cen_vjp_run(tds_b200_sim* s, const float* q, const float* qd, const double* G, double* g_in, double* g_par, cudaStream_t sm) {
  const CenRows R = cen_rows(s);
  const size_t ns = s->ns;
  return vjp_by_eye(s, "centroidal", cen_n_in(s), R.all(), G, g_in, g_par, sm, [&](int nd, const double* t_in, const double* t_par, double* dO) {
    const TdsCenCall out{dO, dO + R.com * nd * ns, dO + (R.com + R.A) * nd * ns};
    return cen_jvp_run(s, q, qd, nd, t_in, t_par, &out, sm);
  });
}

// host q [n][n_q], qd [n][n_qd] (NULL: zero) -> s->q, s->qd; the device pointer of qd (NULL for NULL)
static int put_cen_inputs(tds_b200_sim* s, const double* q, const double* qd, const float** qd_d) {
  int rc = put_q(s, q);
  if (!rc && qd) rc = put_state(s, qd, s->dm[0].n_qd, s->qd);
  *qd_d = qd ? s->qd : nullptr;
  return rc;
}

static int cen_check(tds_b200_sim* s, const void* q, const void* com, const void* A, const void* bias) {
  if (!s || !q || (!com && !A && !bias)) return -1;
  return cen_model_check(s);
}

int tds_b200_centroidal_device(tds_b200_sim* s, const float* q, const float* qd, double* com, double* A, double* bias, void* stream) {
  if (int rc = cen_check(s, q, com, A, bias)) return rc;
  const TdsCenCall out{com, A, bias};
  return cen_run(s, q, qd, &out, (cudaStream_t)stream);
}

int tds_b200_centroidal_host(tds_b200_sim* s, const double* q, const double* qd, double* com, double* A, double* bias) {
  if (int rc = cen_check(s, q, com, A, bias)) return rc;
  if (int rc = enter_derivative_host(s)) return rc;
  const int n = s->n, ns = s->ns;
  const CenRows R = cen_rows(s);
  const float* qd_d;
  if (int rc = put_cen_inputs(s, q, qd, &qd_d)) return rc;
  CUDA_TRY(grow_dev(&s->jac_dev, &s->jac_dev_bytes, sizeof(double) * R.all() * ns));
  double* d = s->jac_dev;
  const TdsCenCall out{com ? d : nullptr, A ? d + R.com * ns : nullptr, bias ? d + (R.com + R.A) * ns : nullptr};
  if (int rc = cen_run(s, s->q, qd_d, &out, s->stream)) return rc;
  CUDA_TRY(get_parts<double>({{com, R.com}, {A, R.A}, {bias, R.bias}}, d, n, ns, s->stream));
  return 0;
}

static int cen_jvp_check(tds_b200_sim* s, const void* q, int m, const void* t_q, const void* t_qd, const void* t_par, const void* t_com,
                         const void* t_A, const void* t_bias) {
  if (!s || !q || m < 1 || (!t_q && !t_qd && !t_par) || (!t_com && !t_A && !t_bias)) return -1;
  if (int rc = cen_model_check(s)) return rc;
  return par_without_installed(s, t_par, "centroidal jvp: parameter tangents");
}

int tds_b200_centroidal_jvp_device(tds_b200_sim* s, const float* q, const float* qd, int m, const double* t_q, const double* t_qd,
                                   const double* t_par, double* t_com, double* t_A, double* t_bias, void* stream) {
  if (int rc = cen_jvp_check(s, q, m, t_q, t_qd, t_par, t_com, t_A, t_bias)) return rc;
  const size_t n_q = s->dm[0].n_q, nd = s->dm[0].n_qd;
  cudaStream_t sm = (cudaStream_t)stream;
  double* tin = nullptr;
  if (t_q || t_qd) {   // the kernel reads the q | qd tangents as one array
    CUDA_TRY(grow_dev(&s->jac_dev, &s->jac_dev_bytes, sizeof(double) * (size_t)cen_n_in(s) * m * s->ns));
    tin = s->jac_dev;
    CUDA_TRY(put_parts_d2d<double>(tin, {{t_q, n_q * m}, {t_qd, nd * m}}, s->ns, sm));
  }
  const TdsCenCall out{t_com, t_A, t_bias};
  return cen_jvp_run(s, q, qd, m, tin, t_par, &out, sm);
}

int tds_b200_centroidal_jvp_host(tds_b200_sim* s, const double* q, const double* qd, int m, const double* t_q, const double* t_qd,
                                 const double* t_par, double* t_com, double* t_A, double* t_bias) {
  if (int rc = cen_jvp_check(s, q, m, t_q, t_qd, t_par, t_com, t_A, t_bias)) return rc;
  if (int rc = enter_derivative_host(s)) return rc;
  const int n = s->n, ns = s->ns;
  const size_t n_q = s->dm[0].n_q, nd = s->dm[0].n_qd;
  const CenRows R = cen_rows(s);
  // tangents: host [n][dim][m] <-> device [dim * m][ns]; q | qd (contiguous, zero where NULL, none if both are), t_par, the outputs
  const size_t ti = (t_q || t_qd) ? (size_t)cen_n_in(s) * m : 0, tp = (size_t)(t_par ? s->par.n : 0) * m;
  const float* qd_d;
  if (int rc = put_cen_inputs(s, q, qd, &qd_d)) return rc;
  CUDA_TRY(grow_dev(&s->jac_dev, &s->jac_dev_bytes, sizeof(double) * (ti + tp + R.all() * m) * ns));
  double* d = s->jac_dev;
  double* to_d = d + (ti + tp) * ns;
  if (ti) CUDA_TRY(put_parts<double>(d, {{t_q, n_q * m}, {t_qd, nd * m}}, n, ns, s->stream));
  if (t_par) CUDA_TRY(put_rows(d + ti * ns, t_par, tp, n, ns, s->stream));
  const TdsCenCall out{t_com ? to_d : nullptr, t_A ? to_d + R.com * m * ns : nullptr, t_bias ? to_d + (R.com + R.A) * m * ns : nullptr};
  if (int rc = cen_jvp_run(s, s->q, qd_d, m, ti ? d : nullptr, t_par ? d + ti * ns : nullptr, &out, s->stream)) return rc;
  CUDA_TRY(get_parts<double>({{t_com, R.com * m}, {t_A, R.A * m}, {t_bias, R.bias * m}}, to_d, n, ns, s->stream));
  return 0;
}

static int cen_vjp_check(tds_b200_sim* s, const void* q, const void* G_com, const void* G_A, const void* G_bias, const void* g_q,
                         const void* g_qd, const void* g_par) {
  if (!s || !q || (!G_com && !G_A && !G_bias) || (!g_q && !g_qd && !g_par)) return -1;
  if (int rc = cen_model_check(s)) return rc;
  return par_without_installed(s, g_par, "centroidal vjp: parameter cotangents");
}

int tds_b200_centroidal_vjp_device(tds_b200_sim* s, const float* q, const float* qd, const double* G_com, const double* G_A,
                                   const double* G_bias, double* g_q, double* g_qd, double* g_par, void* stream) {
  if (int rc = cen_vjp_check(s, q, G_com, G_A, G_bias, g_q, g_qd, g_par)) return rc;
  const size_t n_q = s->dm[0].n_q, nd = s->dm[0].n_qd;
  const CenRows R = cen_rows(s);
  cudaStream_t sm = (cudaStream_t)stream;
  // the concatenated cotangent com | A | bias (zero where a part is NULL), then g_q | g_qd as one array for the contraction
  CUDA_TRY(grow_dev(&s->vjp_g, &s->vjp_g_bytes, sizeof(double) * (R.all() + cen_n_in(s)) * s->ns));
  double* g_d = s->vjp_g + R.all() * s->ns;
  CUDA_TRY(put_parts_d2d<double>(s->vjp_g, {{G_com, R.com}, {G_A, R.A}, {G_bias, R.bias}}, s->ns, sm));
  if (int rc = cen_vjp_run(s, q, qd, s->vjp_g, g_d, g_par, sm)) return rc;
  CUDA_TRY(get_parts_d2d<double>({{g_q, n_q}, {g_qd, nd}}, g_d, s->ns, sm));
  return 0;
}

int tds_b200_centroidal_vjp_host(tds_b200_sim* s, const double* q, const double* qd, const double* G_com, const double* G_A,
                                 const double* G_bias, double* g_q, double* g_qd, double* g_par) {
  if (int rc = cen_vjp_check(s, q, G_com, G_A, G_bias, g_q, g_qd, g_par)) return rc;
  if (int rc = enter_derivative_host(s)) return rc;
  const int n = s->n, ns = s->ns, n_in = cen_n_in(s);
  const size_t n_q = s->dm[0].n_q, nd = s->dm[0].n_qd, k = s->par.n;
  const CenRows R = cen_rows(s);
  const float* qd_d;
  if (int rc = put_cen_inputs(s, q, qd, &qd_d)) return rc;
  // G (com | A | bias, zero where a part is NULL) | g_q | g_qd | g_par
  CUDA_TRY(grow_dev(&s->vjp_g, &s->vjp_g_bytes, sizeof(double) * (R.all() + n_in + k + 1) * ns));
  double* g_d = s->vjp_g + R.all() * ns;
  CUDA_TRY(put_parts<double>(s->vjp_g, {{G_com, R.com}, {G_A, R.A}, {G_bias, R.bias}}, n, ns, s->stream));
  if (int rc = cen_vjp_run(s, s->q, qd_d, s->vjp_g, g_d, g_par ? g_d + (size_t)n_in * ns : nullptr, s->stream)) return rc;
  CUDA_TRY(get_parts<double>({{g_q, n_q}, {g_qd, nd}, {g_par, k}}, g_d, n, ns, s->stream));
  return 0;
}

// ---- derivatives of the inverse dynamics d tau / dq, d tau / dqd (DESIGN.md section 7.23): the DER instances of the world-frame kernel
// (tds_dynamics_derivatives.cu).  The inputs q | qd | qdd are those of the inverse dynamics (inv_n_in, put_inv_inputs). ----------------
// d tau / dq and d tau / dqd [n_qd * n_qd][ns] (either may be NULL) from q [n_q][ns], qd and qdd [n_qd][ns] fp32 (either NULL: zero), or
// at the fp64 qdd64 [n_qd][ns] in place of qdd when that is not NULL (the forward dynamics' derivatives)
static int der_run(tds_b200_sim* s, const float* q, const float* qd, const float* qdd, double* dq, double* dqd, cudaStream_t sm,
                   const double* qdd64 = nullptr) {
  CUDA_TRY(grow_dev(&s->jac_scratch, &s->jac_scratch_bytes, der_arena_bytes(s, s->dm_m, 8)));
  return value_run(s, "inverse dynamics derivatives", q, qd, qdd, dq, [&](const StepIO* io, const ParMap* pm) {
    StepIO d = *io;
    d.g_in = dqd;
    d.g_out = qdd64;
    return tds_launch_dynamics_derivatives(&s->dm_m, &s->P, &d, pm, s->jac_scratch, sm);
  });
}

// t_dq, t_dqd [n_qd * n_qd * m][ns] (either may be NULL) along t_in [(n_q + 2 n_qd) * m][ns] (q | qd | qdd tangents, contiguous) and
// t_par (either may be NULL); dq, dqd, if not NULL, receive the values.  qdd64: as for der_run.
static int der_jvp_run(tds_b200_sim* s, const float* q, const float* qd, const float* qdd, int m, const double* t_in, const double* t_par,
                       double* dq, double* dqd, double* t_dq, double* t_dqd, cudaStream_t sm, const double* qdd64 = nullptr) {
  if (dq || dqd) { if (int rc = der_run(s, q, qd, qdd, dq, dqd, sm, qdd64)) return rc; }
  JvpTangents jv{t_in, t_par, m, Query::der};
  jv.der_dqd = t_dqd;
  jv.der_qdd = qdd64;
  return jacobian_run(s, TDS_B200_MODE_FULL, 0, q, qd, qdd, t_dq, sm, false, &jv);
}

// g_in [(n_q + 2 n_qd)][ns] (q | qd | qdd, contiguous) and g_par [k][ns] (NULL: not wanted) = <G, d(d tau / dq | d tau / dqd)> for the
// cotangent G [2 n_qd^2][ns] of both matrices
static int der_vjp_run(tds_b200_sim* s, const float* q, const float* qd, const float* qdd, const double* G, double* g_in, double* g_par,
                       cudaStream_t sm) {
  const size_t nn = (size_t)s->dm[0].n_qd * s->dm[0].n_qd;
  return vjp_by_eye(s, "inverse dynamics derivatives", inv_n_in(s), 2 * nn, G, g_in, g_par, sm,
                    [&](int nd, const double* t_in, const double* t_par, double* dO) {
                      return der_jvp_run(s, q, qd, qdd, nd, t_in, t_par, nullptr, nullptr, dO, dO + nn * nd * s->ns, sm);
                    });
}

int tds_b200_inverse_dynamics_derivatives_device(tds_b200_sim* s, const float* q, const float* qd, const float* qdd, double* dtau_dq,
                                                 double* dtau_dqd, void* stream) {
  if (!s || !q || (!dtau_dq && !dtau_dqd)) return -1;
  return der_run(s, q, qd, qdd, dtau_dq, dtau_dqd, (cudaStream_t)stream);
}

int tds_b200_inverse_dynamics_derivatives_host(tds_b200_sim* s, const double* q, const double* qd, const double* qdd, double* dtau_dq,
                                               double* dtau_dqd) {
  if (!s || !q || (!dtau_dq && !dtau_dqd)) return -1;
  if (int rc = enter_derivative_host(s)) return rc;
  const size_t nn = (size_t)s->dm[0].n_qd * s->dm[0].n_qd;
  const float *qd_d, *qdd_d;
  if (int rc = put_inv_inputs(s, q, qd, qdd, &qd_d, &qdd_d)) return rc;
  CUDA_TRY(grow_dev(&s->jac_dev, &s->jac_dev_bytes, sizeof(double) * (2 * nn + 1) * s->ns));
  double* d = s->jac_dev;
  if (int rc = der_run(s, s->q, qd_d, qdd_d, dtau_dq ? d : nullptr, dtau_dqd ? d + nn * s->ns : nullptr, s->stream)) return rc;
  CUDA_TRY(get_parts<double>({{dtau_dq, nn}, {dtau_dqd, nn}}, d, s->n, s->ns, s->stream));
  return 0;
}

static int der_jvp_check(tds_b200_sim* s, const void* q, int m, const void* t_q, const void* t_qd, const void* t_qdd, const void* t_par,
                         const void* t_dq, const void* t_dqd) {
  if (!s || !q || (!t_dq && !t_dqd) || m < 1 || (!t_q && !t_qd && !t_qdd && !t_par)) return -1;
  return par_without_installed(s, t_par, "inverse dynamics derivatives jvp: parameter tangents");
}

int tds_b200_inverse_dynamics_derivatives_jvp_device(tds_b200_sim* s, const float* q, const float* qd, const float* qdd, int m,
                                                     const double* t_q, const double* t_qd, const double* t_qdd, const double* t_par,
                                                     double* dtau_dq, double* dtau_dqd, double* t_dtau_dq, double* t_dtau_dqd, void* stream) {
  if (int rc = der_jvp_check(s, q, m, t_q, t_qd, t_qdd, t_par, t_dtau_dq, t_dtau_dqd)) return rc;
  const size_t n_q = s->dm[0].n_q, nd = s->dm[0].n_qd;
  cudaStream_t sm = (cudaStream_t)stream;
  double* tin = nullptr;
  if (t_q || t_qd || t_qdd) {   // the kernel reads the q | qd | qdd tangents as one array
    CUDA_TRY(grow_dev(&s->jac_dev, &s->jac_dev_bytes, sizeof(double) * (size_t)inv_n_in(s) * m * s->ns));
    tin = s->jac_dev;
    CUDA_TRY(put_parts_d2d<double>(tin, {{t_q, n_q * m}, {t_qd, nd * m}, {t_qdd, nd * m}}, s->ns, sm));
  }
  return der_jvp_run(s, q, qd, qdd, m, tin, t_par, dtau_dq, dtau_dqd, t_dtau_dq, t_dtau_dqd, sm);
}

int tds_b200_inverse_dynamics_derivatives_jvp_host(tds_b200_sim* s, const double* q, const double* qd, const double* qdd, int m,
                                                   const double* t_q, const double* t_qd, const double* t_qdd, const double* t_par,
                                                   double* dtau_dq, double* dtau_dqd, double* t_dtau_dq, double* t_dtau_dqd) {
  if (int rc = der_jvp_check(s, q, m, t_q, t_qd, t_qdd, t_par, t_dtau_dq, t_dtau_dqd)) return rc;
  if (int rc = enter_derivative_host(s)) return rc;
  const int n = s->n, ns = s->ns;
  const size_t n_q = s->dm[0].n_q, nd = s->dm[0].n_qd, nn = nd * nd;
  // tangents: host [n][dim][m] <-> device [dim * m][ns]; q | qd | qdd (contiguous, zero where NULL, none if all are), t_par, the
  // tangents of d tau / dq and d tau / dqd, their values
  const size_t ti = (t_q || t_qd || t_qdd) ? (size_t)inv_n_in(s) * m : 0, tp = (size_t)(t_par ? s->par.n : 0) * m, to = nn * m;
  const float *qd_d, *qdd_d;
  if (int rc = put_inv_inputs(s, q, qd, qdd, &qd_d, &qdd_d)) return rc;
  CUDA_TRY(grow_dev(&s->jac_dev, &s->jac_dev_bytes, sizeof(double) * (ti + tp + 2 * to + 2 * nn + 1) * ns));
  double* d = s->jac_dev;
  double* to_d = d + (ti + tp) * ns;
  double* v_d = to_d + 2 * to * ns;
  if (ti) CUDA_TRY(put_parts<double>(d, {{t_q, n_q * m}, {t_qd, nd * m}, {t_qdd, nd * m}}, n, ns, s->stream));
  if (t_par) CUDA_TRY(put_rows(d + ti * ns, t_par, tp, n, ns, s->stream));
  if (int rc = der_jvp_run(s, s->q, qd_d, qdd_d, m, ti ? d : nullptr, t_par ? d + ti * ns : nullptr, dtau_dq ? v_d : nullptr,
                           dtau_dqd ? v_d + nn * ns : nullptr, t_dtau_dq ? to_d : nullptr, t_dtau_dqd ? to_d + to * ns : nullptr, s->stream))
    return rc;
  CUDA_TRY(get_parts<double>({{t_dtau_dq, to}, {t_dtau_dqd, to}, {dtau_dq, nn}, {dtau_dqd, nn}}, to_d, n, ns, s->stream));
  return 0;
}

static int der_vjp_check(tds_b200_sim* s, const void* q, const void* G_dq, const void* G_dqd, const void* g_q, const void* g_qd,
                         const void* g_qdd, const void* g_par) {
  if (!s || !q || (!G_dq && !G_dqd) || (!g_q && !g_qd && !g_qdd && !g_par)) return -1;
  return par_without_installed(s, g_par, "inverse dynamics derivatives vjp: parameter cotangents");
}

int tds_b200_inverse_dynamics_derivatives_vjp_device(tds_b200_sim* s, const float* q, const float* qd, const float* qdd, const double* G_dq,
                                                     const double* G_dqd, double* g_q, double* g_qd, double* g_qdd, double* g_par,
                                                     void* stream) {
  if (int rc = der_vjp_check(s, q, G_dq, G_dqd, g_q, g_qd, g_qdd, g_par)) return rc;
  const size_t n_q = s->dm[0].n_q, nd = s->dm[0].n_qd, nn = nd * nd;
  cudaStream_t sm = (cudaStream_t)stream;
  // the cotangent G_dq | G_dqd (zero where NULL) and g_q | g_qd | g_qdd are one array each: in s->vjp_g, then copied out
  CUDA_TRY(grow_dev(&s->vjp_g, &s->vjp_g_bytes, sizeof(double) * (2 * nn + (size_t)inv_n_in(s)) * s->ns));
  double* g_d = s->vjp_g + 2 * nn * s->ns;
  CUDA_TRY(put_parts_d2d<double>(s->vjp_g, {{G_dq, nn}, {G_dqd, nn}}, s->ns, sm));
  if (int rc = der_vjp_run(s, q, qd, qdd, s->vjp_g, g_d, g_par, sm)) return rc;
  CUDA_TRY(get_parts_d2d<double>({{g_q, n_q}, {g_qd, nd}, {g_qdd, nd}}, g_d, s->ns, sm));
  return 0;
}

int tds_b200_inverse_dynamics_derivatives_vjp_host(tds_b200_sim* s, const double* q, const double* qd, const double* qdd, const double* G_dq,
                                                   const double* G_dqd, double* g_q, double* g_qd, double* g_qdd, double* g_par) {
  if (int rc = der_vjp_check(s, q, G_dq, G_dqd, g_q, g_qd, g_qdd, g_par)) return rc;
  if (int rc = enter_derivative_host(s)) return rc;
  const int n = s->n, ns = s->ns, n_in = inv_n_in(s);
  const size_t n_q = s->dm[0].n_q, nd = s->dm[0].n_qd, nn = nd * nd, k = s->par.n;
  const float *qd_d, *qdd_d;
  if (int rc = put_inv_inputs(s, q, qd, qdd, &qd_d, &qdd_d)) return rc;
  // G_dq | G_dqd | g_q | g_qd | g_qdd | g_par
  CUDA_TRY(grow_dev(&s->vjp_g, &s->vjp_g_bytes, sizeof(double) * (2 * nn + n_in + k + 1) * ns));
  double* g_d = s->vjp_g + 2 * nn * ns;
  CUDA_TRY(put_parts<double>(s->vjp_g, {{G_dq, nn}, {G_dqd, nn}}, n, ns, s->stream));
  if (int rc = der_vjp_run(s, s->q, qd_d, qdd_d, s->vjp_g, g_d, g_par ? g_d + (size_t)n_in * ns : nullptr, s->stream)) return rc;
  CUDA_TRY(get_parts<double>({{g_q, n_q}, {g_qd, nd}, {g_qdd, nd}, {g_par, k}}, g_d, n, ns, s->stream));
  return 0;
}

// ---- Coriolis matrix C(q, qd) (DESIGN.md section 7.22): the COR instances of the world-frame kernel (tds_coriolis.cu).  The inputs
// q | qd are those of the centroidal quantities (cen_n_in, put_cen_inputs). ------------------------------------------------------------
// C [n_qd * n_qd][ns] from q [n_q][ns] and qd [n_qd][ns] fp32 (NULL: zero)
static int cor_run(tds_b200_sim* s, const float* q, const float* qd, double* C, cudaStream_t sm) {
  return value_run(s, "coriolis", q, qd, nullptr, C, [&](const StepIO* io, const ParMap* pm) {
    return tds_launch_coriolis(&s->dm_m, io, pm, s->jac_scratch, sm);
  });
}

// t_C [n_qd * n_qd * m][ns] along t_in [(n_q + n_qd) * m][ns] (q | qd tangents, contiguous) and t_par (either may be NULL); C, if not
// NULL, receives the value
static int cor_jvp_run(tds_b200_sim* s, const float* q, const float* qd, int m, const double* t_in, const double* t_par, double* C, double* t_C,
                       cudaStream_t sm) {
  if (C) { if (int rc = cor_run(s, q, qd, C, sm)) return rc; }
  const JvpTangents jv{t_in, t_par, m, Query::cor};
  return jacobian_run(s, TDS_B200_MODE_FULL, 0, q, qd, nullptr, t_C, sm, false, &jv);
}

// g_in [n_q + n_qd][ns] (q | qd, contiguous) and g_par [k][ns] (NULL: not wanted) = <G, dC>
static int cor_vjp_run(tds_b200_sim* s, const float* q, const float* qd, const double* G, double* g_in, double* g_par, cudaStream_t sm) {
  const size_t nn = (size_t)s->dm[0].n_qd * s->dm[0].n_qd;
  return vjp_by_eye(s, "coriolis", cen_n_in(s), nn, G, g_in, g_par, sm, [&](int nd, const double* t_in, const double* t_par, double* dC) {
    return cor_jvp_run(s, q, qd, nd, t_in, t_par, nullptr, dC, sm);
  });
}

int tds_b200_coriolis_device(tds_b200_sim* s, const float* q, const float* qd, double* C, void* stream) {
  if (!s || !q || !C) return -1;
  return cor_run(s, q, qd, C, (cudaStream_t)stream);
}

int tds_b200_coriolis_host(tds_b200_sim* s, const double* q, const double* qd, double* C) {
  if (!s || !q || !C) return -1;
  if (int rc = enter_derivative_host(s)) return rc;
  const size_t nn = (size_t)s->dm[0].n_qd * s->dm[0].n_qd;
  const float* qd_d;
  if (int rc = put_cen_inputs(s, q, qd, &qd_d)) return rc;
  CUDA_TRY(grow_dev(&s->jac_dev, &s->jac_dev_bytes, sizeof(double) * nn * s->ns));
  if (int rc = cor_run(s, s->q, qd_d, s->jac_dev, s->stream)) return rc;
  CUDA_TRY(get_rows(C, s->jac_dev, nn, s->n, s->ns, s->stream));
  return 0;
}

static int cor_jvp_check(tds_b200_sim* s, const void* q, int m, const void* t_q, const void* t_qd, const void* t_par, const void* t_C) {
  if (!s || !q || !t_C || m < 1 || (!t_q && !t_qd && !t_par)) return -1;
  return par_without_installed(s, t_par, "coriolis jvp: parameter tangents");
}

int tds_b200_coriolis_jvp_device(tds_b200_sim* s, const float* q, const float* qd, int m, const double* t_q, const double* t_qd,
                                 const double* t_par, double* C, double* t_C, void* stream) {
  if (int rc = cor_jvp_check(s, q, m, t_q, t_qd, t_par, t_C)) return rc;
  const size_t n_q = s->dm[0].n_q, nd = s->dm[0].n_qd;
  cudaStream_t sm = (cudaStream_t)stream;
  double* tin = nullptr;
  if (t_q || t_qd) {   // the kernel reads the q | qd tangents as one array
    CUDA_TRY(grow_dev(&s->jac_dev, &s->jac_dev_bytes, sizeof(double) * (size_t)cen_n_in(s) * m * s->ns));
    tin = s->jac_dev;
    CUDA_TRY(put_parts_d2d<double>(tin, {{t_q, n_q * m}, {t_qd, nd * m}}, s->ns, sm));
  }
  return cor_jvp_run(s, q, qd, m, tin, t_par, C, t_C, sm);
}

int tds_b200_coriolis_jvp_host(tds_b200_sim* s, const double* q, const double* qd, int m, const double* t_q, const double* t_qd,
                               const double* t_par, double* C, double* t_C) {
  if (int rc = cor_jvp_check(s, q, m, t_q, t_qd, t_par, t_C)) return rc;
  if (int rc = enter_derivative_host(s)) return rc;
  const int n = s->n, ns = s->ns;
  const size_t n_q = s->dm[0].n_q, nd = s->dm[0].n_qd, nn = nd * nd;
  // tangents: host [n][dim][m] <-> device [dim * m][ns]; q | qd (contiguous, zero where NULL, none if both are), t_par, t_C, C
  const size_t ti = (t_q || t_qd) ? (size_t)cen_n_in(s) * m : 0, tp = (size_t)(t_par ? s->par.n : 0) * m, to = nn * m;
  const float* qd_d;
  if (int rc = put_cen_inputs(s, q, qd, &qd_d)) return rc;
  CUDA_TRY(grow_dev(&s->jac_dev, &s->jac_dev_bytes, sizeof(double) * (ti + tp + to + nn) * ns));
  double* d = s->jac_dev;
  double* to_d = d + (ti + tp) * ns;
  if (ti) CUDA_TRY(put_parts<double>(d, {{t_q, n_q * m}, {t_qd, nd * m}}, n, ns, s->stream));
  if (t_par) CUDA_TRY(put_rows(d + ti * ns, t_par, tp, n, ns, s->stream));
  if (int rc = cor_jvp_run(s, s->q, qd_d, m, ti ? d : nullptr, t_par ? d + ti * ns : nullptr, C ? to_d + to * ns : nullptr, to_d, s->stream))
    return rc;
  CUDA_TRY(get_parts<double>({{t_C, to}, {C, nn}}, to_d, n, ns, s->stream));
  return 0;
}

static int cor_vjp_check(tds_b200_sim* s, const void* q, const void* G, const void* g_q, const void* g_qd, const void* g_par) {
  if (!s || !q || !G || (!g_q && !g_qd && !g_par)) return -1;
  return par_without_installed(s, g_par, "coriolis vjp: parameter cotangents");
}

int tds_b200_coriolis_vjp_device(tds_b200_sim* s, const float* q, const float* qd, const double* G, double* g_q, double* g_qd, double* g_par,
                                 void* stream) {
  if (int rc = cor_vjp_check(s, q, G, g_q, g_qd, g_par)) return rc;
  const size_t n_q = s->dm[0].n_q, nd = s->dm[0].n_qd;
  cudaStream_t sm = (cudaStream_t)stream;
  // g_q | g_qd are one array for the contraction: computed in s->vjp_g, then copied out
  CUDA_TRY(grow_dev(&s->vjp_g, &s->vjp_g_bytes, sizeof(double) * (size_t)cen_n_in(s) * s->ns));
  if (int rc = cor_vjp_run(s, q, qd, G, s->vjp_g, g_par, sm)) return rc;
  CUDA_TRY(get_parts_d2d<double>({{g_q, n_q}, {g_qd, nd}}, s->vjp_g, s->ns, sm));
  return 0;
}

int tds_b200_coriolis_vjp_host(tds_b200_sim* s, const double* q, const double* qd, const double* G, double* g_q, double* g_qd, double* g_par) {
  if (int rc = cor_vjp_check(s, q, G, g_q, g_qd, g_par)) return rc;
  if (int rc = enter_derivative_host(s)) return rc;
  const int n = s->n, ns = s->ns, n_in = cen_n_in(s);
  const size_t n_q = s->dm[0].n_q, nd = s->dm[0].n_qd, nn = nd * nd, k = s->par.n;
  const float* qd_d;
  if (int rc = put_cen_inputs(s, q, qd, &qd_d)) return rc;
  // G | g_q | g_qd | g_par
  CUDA_TRY(grow_dev(&s->vjp_g, &s->vjp_g_bytes, sizeof(double) * (nn + n_in + k + 1) * ns));
  double* g_d = s->vjp_g + nn * ns;
  CUDA_TRY(put_rows(s->vjp_g, G, nn, n, ns, s->stream));
  if (int rc = cor_vjp_run(s, s->q, qd_d, s->vjp_g, g_d, g_par ? g_d + (size_t)n_in * ns : nullptr, s->stream)) return rc;
  CUDA_TRY(get_parts<double>({{g_q, n_q}, {g_qd, nd}, {g_par, k}}, g_d, n, ns, s->stream));
  return 0;
}

// ---- spatial point Jacobians, point velocities and accelerations (DESIGN.md section 7.17): the MOT instances of the world-frame kernel
// (tds_point_motion.cu).  The point table is checked as for the kinematics (kin_check); the inputs q | qd | qdd are those of inverse
// dynamics (inv_n_in, put_inv_inputs). -----------------------------------------------------------------------------------------------------
// rows of the outputs J | vel | acc
struct MotRows { size_t J, vel, acc; size_t all() const { return J + vel + acc; } };
static MotRows mot_rows(const tds_b200_sim* s, int K) { return MotRows{(size_t)6 * K * s->dm[0].n_qd, (size_t)6 * K, (size_t)6 * K}; }

// fp64 outputs from q [n_q][ns], qd and qdd [n_qd][ns] fp32 (either NULL: zero; installed parameters do not enter)
static int mot_run(tds_b200_sim* s, const float* q, const float* qd, const float* qdd, const TdsMotCall* mc, cudaStream_t sm) {
  return value_run(s, "point motion", q, qd, qdd, nullptr, [&](const StepIO* io, const ParMap*) {
    return tds_launch_point_motion(&s->dm_m, io, mc, s->jac_scratch, sm);
  });
}

// m tangents t_in [(n_q + 2 n_qd) * m][ns] (q | qd | qdd, contiguous) -> the outputs' columns [rows * m][ns], through the Jacobian's chunk
// loop
static int mot_jvp_run(tds_b200_sim* s, const float* q, const float* qd, const float* qdd, const TdsMotCall* mc, int m, const double* t_in,
                       cudaStream_t sm) {
  JvpTangents jv{t_in, nullptr, m, Query::motion};
  jv.mot = mc;
  return jacobian_run(s, TDS_B200_MODE_FULL, 0, q, qd, qdd, nullptr, sm, false, &jv);
}

// g_in [n_q + 2 n_qd][ns] (q | qd | qdd, contiguous) = <G, d(J | vel | acc)>, G [rows][ns] concatenated
static int mot_vjp_run(tds_b200_sim* s, const float* q, const float* qd, const float* qdd, int K, const int* links, const double* local,
                       const double* G, double* g_in, cudaStream_t sm) {
  const MotRows R = mot_rows(s, K);
  const size_t ns = s->ns;
  return vjp_by_eye(s, "point motion", inv_n_in(s), R.all(), G, g_in, nullptr, sm, [&](int nd, const double* t_in, const double*, double* dO) {
    const TdsMotCall mc{K, links, local, dO, dO + R.J * nd * ns, dO + (R.J + R.vel) * nd * ns};
    return mot_jvp_run(s, q, qd, qdd, &mc, nd, t_in, sm);
  });
}

static int mot_check(tds_b200_sim* s, const void* q, int K, const int* links, const double* local, const void* J, const void* vel,
                     const void* acc) {
  if (int rc = kin_check(s, q, K, links, local)) return rc;
  if (!J && !vel && !acc) return -1;
  return 0;
}

int tds_b200_point_motion_device(tds_b200_sim* s, const float* q, const float* qd, const float* qdd, int K, const int* links,
                                 const double* local, double* J, double* vel, double* acc, void* stream) {
  if (int rc = mot_check(s, q, K, links, local, J, vel, acc)) return rc;
  const TdsMotCall mc{K, links, local, J, vel, acc};
  return mot_run(s, q, qd, qdd, &mc, (cudaStream_t)stream);
}

int tds_b200_point_motion_host(tds_b200_sim* s, const double* q, const double* qd, const double* qdd, int K, const int* links,
                               const double* local, double* J, double* vel, double* acc) {
  if (int rc = mot_check(s, q, K, links, local, J, vel, acc)) return rc;
  if (int rc = enter_derivative_host(s)) return rc;
  const int n = s->n, ns = s->ns;
  const MotRows R = mot_rows(s, K);
  const float *qd_d, *qdd_d;
  if (int rc = put_inv_inputs(s, q, qd, qdd, &qd_d, &qdd_d)) return rc;
  CUDA_TRY(grow_dev(&s->jac_dev, &s->jac_dev_bytes, sizeof(double) * (R.all() + 1) * ns));
  double* d = s->jac_dev;
  const TdsMotCall mc{K, links, local, J ? d : nullptr, vel ? d + R.J * ns : nullptr, acc ? d + (R.J + R.vel) * ns : nullptr};
  if (int rc = mot_run(s, s->q, qd_d, qdd_d, &mc, s->stream)) return rc;
  CUDA_TRY(get_parts<double>({{J, R.J}, {vel, R.vel}, {acc, R.acc}}, d, n, ns, s->stream));
  return 0;
}

static int mot_jvp_check(tds_b200_sim* s, const void* q, int K, const int* links, const double* local, int m, const void* t_q,
                         const void* t_qd, const void* t_qdd, const void* t_J, const void* t_vel, const void* t_acc) {
  if (int rc = mot_check(s, q, K, links, local, t_J, t_vel, t_acc)) return rc;
  if (m < 1 || (!t_q && !t_qd && !t_qdd)) return -1;
  return 0;
}

int tds_b200_point_motion_jvp_device(tds_b200_sim* s, const float* q, const float* qd, const float* qdd, int K, const int* links,
                                     const double* local, int m, const double* t_q, const double* t_qd, const double* t_qdd, double* t_J,
                                     double* t_vel, double* t_acc, void* stream) {
  if (int rc = mot_jvp_check(s, q, K, links, local, m, t_q, t_qd, t_qdd, t_J, t_vel, t_acc)) return rc;
  const size_t n_q = s->dm[0].n_q, nd = s->dm[0].n_qd;
  cudaStream_t sm = (cudaStream_t)stream;
  // the kernel reads the q | qd | qdd tangents as one array
  CUDA_TRY(grow_dev(&s->jac_dev, &s->jac_dev_bytes, sizeof(double) * (size_t)inv_n_in(s) * m * s->ns));
  double* tin = s->jac_dev;
  CUDA_TRY(put_parts_d2d<double>(tin, {{t_q, n_q * m}, {t_qd, nd * m}, {t_qdd, nd * m}}, s->ns, sm));
  const TdsMotCall mc{K, links, local, t_J, t_vel, t_acc};
  return mot_jvp_run(s, q, qd, qdd, &mc, m, tin, sm);
}

int tds_b200_point_motion_jvp_host(tds_b200_sim* s, const double* q, const double* qd, const double* qdd, int K, const int* links,
                                   const double* local, int m, const double* t_q, const double* t_qd, const double* t_qdd, double* t_J,
                                   double* t_vel, double* t_acc) {
  if (int rc = mot_jvp_check(s, q, K, links, local, m, t_q, t_qd, t_qdd, t_J, t_vel, t_acc)) return rc;
  if (int rc = enter_derivative_host(s)) return rc;
  const int n = s->n, ns = s->ns;
  const size_t n_q = s->dm[0].n_q, nd = s->dm[0].n_qd;
  const MotRows R = mot_rows(s, K);
  // tangents: host [n][dim][m] <-> device [dim * m][ns]; q | qd | qdd (contiguous, zero where NULL), then the outputs
  const size_t ti = (size_t)inv_n_in(s) * m;
  const float *qd_d, *qdd_d;
  if (int rc = put_inv_inputs(s, q, qd, qdd, &qd_d, &qdd_d)) return rc;
  CUDA_TRY(grow_dev(&s->jac_dev, &s->jac_dev_bytes, sizeof(double) * (ti + R.all() * m + 1) * ns));
  double* d = s->jac_dev;
  double* to_d = d + ti * ns;
  CUDA_TRY(put_parts<double>(d, {{t_q, n_q * m}, {t_qd, nd * m}, {t_qdd, nd * m}}, n, ns, s->stream));
  const TdsMotCall mc{K, links, local, t_J ? to_d : nullptr, t_vel ? to_d + R.J * m * ns : nullptr,
                      t_acc ? to_d + (R.J + R.vel) * m * ns : nullptr};
  if (int rc = mot_jvp_run(s, s->q, qd_d, qdd_d, &mc, m, d, s->stream)) return rc;
  CUDA_TRY(get_parts<double>({{t_J, R.J * m}, {t_vel, R.vel * m}, {t_acc, R.acc * m}}, to_d, n, ns, s->stream));
  return 0;
}

static int mot_vjp_check(tds_b200_sim* s, const void* q, int K, const int* links, const double* local, const void* G_J, const void* G_vel,
                         const void* G_acc, const void* g_q, const void* g_qd, const void* g_qdd) {
  if (int rc = mot_check(s, q, K, links, local, G_J, G_vel, G_acc)) return rc;
  if (!g_q && !g_qd && !g_qdd) return -1;
  return 0;
}

int tds_b200_point_motion_vjp_device(tds_b200_sim* s, const float* q, const float* qd, const float* qdd, int K, const int* links,
                                     const double* local, const double* G_J, const double* G_vel, const double* G_acc, double* g_q,
                                     double* g_qd, double* g_qdd, void* stream) {
  if (int rc = mot_vjp_check(s, q, K, links, local, G_J, G_vel, G_acc, g_q, g_qd, g_qdd)) return rc;
  const size_t n_q = s->dm[0].n_q, nd = s->dm[0].n_qd;
  const MotRows R = mot_rows(s, K);
  cudaStream_t sm = (cudaStream_t)stream;
  // the concatenated cotangent J | vel | acc (zero where a part is NULL), then g_q | g_qd | g_qdd as one array for the contraction
  CUDA_TRY(grow_dev(&s->vjp_g, &s->vjp_g_bytes, sizeof(double) * (R.all() + inv_n_in(s)) * s->ns));
  double* g_d = s->vjp_g + R.all() * s->ns;
  CUDA_TRY(put_parts_d2d<double>(s->vjp_g, {{G_J, R.J}, {G_vel, R.vel}, {G_acc, R.acc}}, s->ns, sm));
  if (int rc = mot_vjp_run(s, q, qd, qdd, K, links, local, s->vjp_g, g_d, sm)) return rc;
  CUDA_TRY(get_parts_d2d<double>({{g_q, n_q}, {g_qd, nd}, {g_qdd, nd}}, g_d, s->ns, sm));
  return 0;
}

int tds_b200_point_motion_vjp_host(tds_b200_sim* s, const double* q, const double* qd, const double* qdd, int K, const int* links,
                                   const double* local, const double* G_J, const double* G_vel, const double* G_acc, double* g_q,
                                   double* g_qd, double* g_qdd) {
  if (int rc = mot_vjp_check(s, q, K, links, local, G_J, G_vel, G_acc, g_q, g_qd, g_qdd)) return rc;
  if (int rc = enter_derivative_host(s)) return rc;
  const int n = s->n, ns = s->ns;
  const size_t n_q = s->dm[0].n_q, nd = s->dm[0].n_qd;
  const MotRows R = mot_rows(s, K);
  const float *qd_d, *qdd_d;
  if (int rc = put_inv_inputs(s, q, qd, qdd, &qd_d, &qdd_d)) return rc;
  // G (J | vel | acc, zero where a part is NULL) | g_q | g_qd | g_qdd
  CUDA_TRY(grow_dev(&s->vjp_g, &s->vjp_g_bytes, sizeof(double) * (R.all() + inv_n_in(s)) * ns));
  double* g_d = s->vjp_g + R.all() * ns;
  CUDA_TRY(put_parts<double>(s->vjp_g, {{G_J, R.J}, {G_vel, R.vel}, {G_acc, R.acc}}, n, ns, s->stream));
  if (int rc = mot_vjp_run(s, s->q, qd_d, qdd_d, K, links, local, s->vjp_g, g_d, s->stream)) return rc;
  CUDA_TRY(get_parts<double>({{g_q, n_q}, {g_qd, nd}, {g_qdd, nd}}, g_d, n, ns, s->stream));
  return 0;
}

// ---- joint-torque and energy regressors of the inertial parameters (DESIGN.md section 7.19): the REG instances of the world-frame kernel
// (tds_regressor.cu).  The inputs q | qd | qdd are those of inverse dynamics (inv_n_in, put_inv_inputs). ----------------------------------
// rows of the outputs Y | yT | yV, with n_pi = 12 n_links + 10 parameter columns (the physical-parameter ids from 2 on)
struct RegRows { size_t Y, yT, yV; size_t all() const { return Y + yT + yV; } };
static RegRows reg_rows(const tds_b200_sim* s) {
  const size_t n_pi = (size_t)12 * s->dm[0].n_links + 10;
  return RegRows{(size_t)s->dm[0].n_qd * n_pi, n_pi, n_pi};
}

// fp64 Y [n_qd * n_pi][ns] and out->yT, out->yV [n_pi][ns] (each may be NULL) from q [n_q][ns], qd and qdd [n_qd][ns] fp32 (either NULL:
// zero; installed parameters do not enter)
static int reg_run(tds_b200_sim* s, const float* q, const float* qd, const float* qdd, double* Y, const TdsRegCall* out, cudaStream_t sm) {
  return value_run(s, "regressor", q, qd, qdd, Y, [&](const StepIO* io, const ParMap*) {
    return tds_launch_regressor(&s->dm_m, &s->P, io, out, s->jac_scratch, sm);
  });
}

// m tangents t_in [(n_q + 2 n_qd) * m][ns] (q | qd | qdd, contiguous) -> the outputs' columns t_Y [R.Y * m][ns], out->yT and out->yV
// [n_pi * m][ns], through the Jacobian's chunk loop
static int reg_jvp_run(tds_b200_sim* s, const float* q, const float* qd, const float* qdd, const TdsRegCall* out, int m, const double* t_in,
                       double* t_Y, cudaStream_t sm) {
  JvpTangents jv{t_in, nullptr, m, Query::regressor};
  jv.reg = out;
  return jacobian_run(s, TDS_B200_MODE_FULL, 0, q, qd, qdd, t_Y, sm, false, &jv);
}

// g_in [n_q + 2 n_qd][ns] (q | qd | qdd, contiguous) = <G, d(Y | yT | yV)>, G [rows][ns] concatenated
static int reg_vjp_run(tds_b200_sim* s, const float* q, const float* qd, const float* qdd, const double* G, double* g_in, cudaStream_t sm) {
  const RegRows R = reg_rows(s);
  const size_t ns = s->ns;
  return vjp_by_eye(s, "regressor", inv_n_in(s), R.all(), G, g_in, nullptr, sm, [&](int nd, const double* t_in, const double*, double* dO) {
    const TdsRegCall out{dO + R.Y * nd * ns, dO + (R.Y + R.yT) * nd * ns};
    return reg_jvp_run(s, q, qd, qdd, &out, nd, t_in, dO, sm);
  });
}

static int reg_check(tds_b200_sim* s, const void* q, const void* Y, const void* yT, const void* yV) {
  if (!s || !q || (!Y && !yT && !yV)) return -1;
  return 0;
}

int tds_b200_regressor_device(tds_b200_sim* s, const float* q, const float* qd, const float* qdd, double* Y, double* yT, double* yV,
                              void* stream) {
  if (int rc = reg_check(s, q, Y, yT, yV)) return rc;
  const TdsRegCall out{yT, yV};
  return reg_run(s, q, qd, qdd, Y, &out, (cudaStream_t)stream);
}

int tds_b200_regressor_host(tds_b200_sim* s, const double* q, const double* qd, const double* qdd, double* Y, double* yT, double* yV) {
  if (int rc = reg_check(s, q, Y, yT, yV)) return rc;
  if (int rc = enter_derivative_host(s)) return rc;
  const int n = s->n, ns = s->ns;
  const RegRows R = reg_rows(s);
  const float *qd_d, *qdd_d;
  if (int rc = put_inv_inputs(s, q, qd, qdd, &qd_d, &qdd_d)) return rc;
  CUDA_TRY(grow_dev(&s->jac_dev, &s->jac_dev_bytes, sizeof(double) * (R.all() + 1) * ns));
  double* d = s->jac_dev;
  const TdsRegCall out{yT ? d + R.Y * ns : nullptr, yV ? d + (R.Y + R.yT) * ns : nullptr};
  if (int rc = reg_run(s, s->q, qd_d, qdd_d, Y ? d : nullptr, &out, s->stream)) return rc;
  CUDA_TRY(get_parts<double>({{Y, R.Y}, {yT, R.yT}, {yV, R.yV}}, d, n, ns, s->stream));
  return 0;
}

static int reg_jvp_check(tds_b200_sim* s, const void* q, int m, const void* t_q, const void* t_qd, const void* t_qdd, const void* t_Y,
                         const void* t_yT, const void* t_yV) {
  if (int rc = reg_check(s, q, t_Y, t_yT, t_yV)) return rc;
  if (m < 1 || (!t_q && !t_qd && !t_qdd)) return -1;
  return 0;
}

int tds_b200_regressor_jvp_device(tds_b200_sim* s, const float* q, const float* qd, const float* qdd, int m, const double* t_q,
                                  const double* t_qd, const double* t_qdd, double* t_Y, double* t_yT, double* t_yV, void* stream) {
  if (int rc = reg_jvp_check(s, q, m, t_q, t_qd, t_qdd, t_Y, t_yT, t_yV)) return rc;
  const size_t n_q = s->dm[0].n_q, nd = s->dm[0].n_qd;
  cudaStream_t sm = (cudaStream_t)stream;
  // the kernel reads the q | qd | qdd tangents as one array
  CUDA_TRY(grow_dev(&s->jac_dev, &s->jac_dev_bytes, sizeof(double) * (size_t)inv_n_in(s) * m * s->ns));
  double* tin = s->jac_dev;
  CUDA_TRY(put_parts_d2d<double>(tin, {{t_q, n_q * m}, {t_qd, nd * m}, {t_qdd, nd * m}}, s->ns, sm));
  const TdsRegCall out{t_yT, t_yV};
  return reg_jvp_run(s, q, qd, qdd, &out, m, tin, t_Y, sm);
}

int tds_b200_regressor_jvp_host(tds_b200_sim* s, const double* q, const double* qd, const double* qdd, int m, const double* t_q,
                                const double* t_qd, const double* t_qdd, double* t_Y, double* t_yT, double* t_yV) {
  if (int rc = reg_jvp_check(s, q, m, t_q, t_qd, t_qdd, t_Y, t_yT, t_yV)) return rc;
  if (int rc = enter_derivative_host(s)) return rc;
  const int n = s->n, ns = s->ns;
  const size_t n_q = s->dm[0].n_q, nd = s->dm[0].n_qd;
  const RegRows R = reg_rows(s);
  // tangents: host [n][dim][m] <-> device [dim * m][ns]; q | qd | qdd (contiguous, zero where NULL), then the outputs
  const size_t ti = (size_t)inv_n_in(s) * m;
  const float *qd_d, *qdd_d;
  if (int rc = put_inv_inputs(s, q, qd, qdd, &qd_d, &qdd_d)) return rc;
  CUDA_TRY(grow_dev(&s->jac_dev, &s->jac_dev_bytes, sizeof(double) * (ti + R.all() * m + 1) * ns));
  double* d = s->jac_dev;
  double* to_d = d + ti * ns;
  CUDA_TRY(put_parts<double>(d, {{t_q, n_q * m}, {t_qd, nd * m}, {t_qdd, nd * m}}, n, ns, s->stream));
  const TdsRegCall out{t_yT ? to_d + R.Y * m * ns : nullptr, t_yV ? to_d + (R.Y + R.yT) * m * ns : nullptr};
  if (int rc = reg_jvp_run(s, s->q, qd_d, qdd_d, &out, m, d, t_Y ? to_d : nullptr, s->stream)) return rc;
  CUDA_TRY(get_parts<double>({{t_Y, R.Y * m}, {t_yT, R.yT * m}, {t_yV, R.yV * m}}, to_d, n, ns, s->stream));
  return 0;
}

static int reg_vjp_check(tds_b200_sim* s, const void* q, const void* G_Y, const void* G_yT, const void* G_yV, const void* g_q,
                         const void* g_qd, const void* g_qdd) {
  if (int rc = reg_check(s, q, G_Y, G_yT, G_yV)) return rc;
  if (!g_q && !g_qd && !g_qdd) return -1;
  return 0;
}

int tds_b200_regressor_vjp_device(tds_b200_sim* s, const float* q, const float* qd, const float* qdd, const double* G_Y, const double* G_yT,
                                  const double* G_yV, double* g_q, double* g_qd, double* g_qdd, void* stream) {
  if (int rc = reg_vjp_check(s, q, G_Y, G_yT, G_yV, g_q, g_qd, g_qdd)) return rc;
  const size_t n_q = s->dm[0].n_q, nd = s->dm[0].n_qd;
  const RegRows R = reg_rows(s);
  cudaStream_t sm = (cudaStream_t)stream;
  // the concatenated cotangent Y | yT | yV (zero where a part is NULL), then g_q | g_qd | g_qdd as one array for the contraction
  CUDA_TRY(grow_dev(&s->vjp_g, &s->vjp_g_bytes, sizeof(double) * (R.all() + inv_n_in(s)) * s->ns));
  double* g_d = s->vjp_g + R.all() * s->ns;
  CUDA_TRY(put_parts_d2d<double>(s->vjp_g, {{G_Y, R.Y}, {G_yT, R.yT}, {G_yV, R.yV}}, s->ns, sm));
  if (int rc = reg_vjp_run(s, q, qd, qdd, s->vjp_g, g_d, sm)) return rc;
  CUDA_TRY(get_parts_d2d<double>({{g_q, n_q}, {g_qd, nd}, {g_qdd, nd}}, g_d, s->ns, sm));
  return 0;
}

int tds_b200_regressor_vjp_host(tds_b200_sim* s, const double* q, const double* qd, const double* qdd, const double* G_Y, const double* G_yT,
                                const double* G_yV, double* g_q, double* g_qd, double* g_qdd) {
  if (int rc = reg_vjp_check(s, q, G_Y, G_yT, G_yV, g_q, g_qd, g_qdd)) return rc;
  if (int rc = enter_derivative_host(s)) return rc;
  const int n = s->n, ns = s->ns;
  const size_t n_q = s->dm[0].n_q, nd = s->dm[0].n_qd;
  const RegRows R = reg_rows(s);
  const float *qd_d, *qdd_d;
  if (int rc = put_inv_inputs(s, q, qd, qdd, &qd_d, &qdd_d)) return rc;
  // G (Y | yT | yV, zero where a part is NULL) | g_q | g_qd | g_qdd
  CUDA_TRY(grow_dev(&s->vjp_g, &s->vjp_g_bytes, sizeof(double) * (R.all() + inv_n_in(s)) * ns));
  double* g_d = s->vjp_g + R.all() * ns;
  CUDA_TRY(put_parts<double>(s->vjp_g, {{G_Y, R.Y}, {G_yT, R.yT}, {G_yV, R.yV}}, n, ns, s->stream));
  if (int rc = reg_vjp_run(s, s->q, qd_d, qdd_d, s->vjp_g, g_d, s->stream)) return rc;
  CUDA_TRY(get_parts<double>({{g_q, n_q}, {g_qd, nd}, {g_qdd, nd}}, g_d, n, ns, s->stream));
  return 0;
}

// ---- inverse mass matrix M^-1(q) and operational-space inverse inertia J M^-1 J^T (DESIGN.md section 7.20): the MINV instances of the
// world-frame kernel and the contraction kernel (tds_mass_inverse.cu), with J from the point-motion value and JVP (mot_run, mot_jvp_run) --
// rows of the outputs M^-1 | Lambda^-1
struct MinvRows { size_t Mi, L; size_t all() const { return Mi + L; } };
static MinvRows minv_rows(const tds_b200_sim* s, int K) {
  return MinvRows{(size_t)s->dm[0].n_qd * s->dm[0].n_qd, (size_t)36 * K * K};
}

// M^-1 [nn][ns] and Lambda^-1 [36 K^2][ns] (either may be null) from q [n_q][ns] fp32 and, with m tangents t_q [n_q * m][ns] and t_par
// [k * m][ns] (either may be null: zero), their tangents t_Minv [nn * m][ns] and t_Linv [36 K^2 * m][ns] (either may be null).  What the
// outputs need and the caller does not ask for (M^-1 and its tangents, J and dJ, the q | qd | qdd tangents of the point-motion JVP) goes
// to s->minv_dev.
static int minv_run(tds_b200_sim* s, const float* q, int K, const int* links, const double* local, double* Minv, double* Linv, int m,
                    const double* t_q, const double* t_par, double* t_Minv, double* t_Linv, cudaStream_t sm) {
  const DevModel& D = s->dm[0];
  const size_t ns = s->ns, nn = (size_t)D.n_qd * D.n_qd, nJ = (size_t)6 * K * D.n_qd;
  const bool lam = Linv || t_Linv, dlam_q = t_Linv && t_q;
  const size_t sMi = (lam && !Minv) ? nn : 0, sJ = lam ? nJ : 0, sdMi = (t_Linv && !t_Minv) ? nn * m : 0, sdJ = dlam_q ? nJ * m : 0,
               sT = dlam_q ? (size_t)inv_n_in(s) * m : 0;
  CUDA_TRY(grow_dev(&s->minv_dev, &s->minv_dev_bytes, sizeof(double) * (sMi + sJ + sdMi + sdJ + sT + 1) * ns));
  double* const Mi = Minv ? Minv : s->minv_dev;
  double* const J = s->minv_dev + sMi * ns;
  double* const dMi = t_Minv ? t_Minv : J + sJ * ns;
  double* const dJ = J + (sJ + sdMi) * ns;
  double* const T = dJ + sdJ * ns;
  if (Minv || lam) {
    int rc = value_run(s, "mass inverse", q, nullptr, nullptr, Mi, [&](const StepIO* io, const ParMap* pm) {
      return tds_launch_mass_inverse(&s->dm_m, io, pm, s->jac_scratch, sm);
    });
    if (rc) return rc;
  }
  const TdsMotCall mc{K, links, local, J, nullptr, nullptr}, dmc{K, links, local, dJ, nullptr, nullptr};
  if (lam) { if (int rc = mot_run(s, q, nullptr, nullptr, &mc, sm)) return rc; }
  if (t_Minv || t_Linv) {
    const JvpTangents jv{t_q, t_par, m, Query::minv};
    if (int rc = jacobian_run(s, TDS_B200_MODE_FULL, 0, q, nullptr, nullptr, dMi, sm, false, &jv)) return rc;
    if (dlam_q) {   // J depends on q alone: its tangents along the q tangents (qd and qdd tangents zero)
      CUDA_TRY(put_parts_d2d<double>(T, {{t_q, (size_t)D.n_q * m}, {nullptr, (size_t)2 * D.n_qd * m}}, s->ns, sm));
      if (int rc = mot_jvp_run(s, q, nullptr, nullptr, &dmc, m, T, sm)) return rc;
    }
  }
  int rc = 0;
  if (Linv) rc = tds_launch_osim(J, nullptr, Mi, nullptr, Linv, K, D.n_qd, 1, s->n, s->ns, sm);
  if (!rc && t_Linv) rc = tds_launch_osim(J, dlam_q ? dJ : nullptr, Mi, dMi, t_Linv, K, D.n_qd, m, s->n, s->ns, sm);
  if (rc) set_err(std::string("mass inverse: J M^-1 J^T launch: ") + cudaGetErrorString((cudaError_t)rc));
  return rc;
}

// g_q [n_q][ns] and g_par [k][ns] (either may be null) = <G, d(M^-1 | Lambda^-1)>, G [nn + 36 K^2][ns] concatenated, or G [nn][ns] alone
// when with_L is false
static int minv_vjp_run(tds_b200_sim* s, const float* q, int K, const int* links, const double* local, bool with_L, const double* G,
                        double* g_q, double* g_par, cudaStream_t sm) {
  const MinvRows R = minv_rows(s, K);
  const size_t ns = s->ns;
  return vjp_by_eye(s, "mass inverse", s->dm[0].n_q, R.Mi + (with_L ? R.L : 0), G, g_q, g_par, sm,
                    [&](int nd, const double* t_q, const double* t_par, double* dO) {
                      return minv_run(s, q, K, links, local, nullptr, nullptr, nd, t_q, t_par, dO, with_L ? dO + R.Mi * nd * ns : nullptr,
                                      sm);
                    });
}

// -1: no q, no output (Minv, Linv), K out of [0, TDS_B200_MAX_OSIM_POINTS], Linv with K = 0, a missing or bad point table
static int minv_check(tds_b200_sim* s, const void* q, int K, const int* links, const double* local, const void* Minv, const void* Linv) {
  if (!s || !q || (!Minv && !Linv)) return -1;
  if (K < 0 || K > TDS_B200_MAX_OSIM_POINTS) { set_err("mass inverse: K out of [0, TDS_B200_MAX_OSIM_POINTS]"); return -1; }
  if (Linv && K < 1) { set_err("mass inverse: J M^-1 J^T needs K >= 1 points"); return -1; }
  return kin_check(s, q, K, links, local);
}

int tds_b200_mass_inverse_device(tds_b200_sim* s, const float* q, int K, const int* links, const double* local, double* Minv, double* Linv,
                                 void* stream) {
  if (int rc = minv_check(s, q, K, links, local, Minv, Linv)) return rc;
  return minv_run(s, q, K, links, local, Minv, Linv, 0, nullptr, nullptr, nullptr, nullptr, (cudaStream_t)stream);
}

int tds_b200_mass_inverse_host(tds_b200_sim* s, const double* q, int K, const int* links, const double* local, double* Minv, double* Linv) {
  if (int rc = minv_check(s, q, K, links, local, Minv, Linv)) return rc;
  if (int rc = enter_derivative_host(s)) return rc;
  const int n = s->n, ns = s->ns;
  const MinvRows R = minv_rows(s, K);
  if (int rc = put_q(s, q)) return rc;
  CUDA_TRY(grow_dev(&s->jac_dev, &s->jac_dev_bytes, sizeof(double) * (R.all() + 1) * ns));
  double* d = s->jac_dev;
  if (int rc = minv_run(s, s->q, K, links, local, Minv ? d : nullptr, Linv ? d + R.Mi * ns : nullptr, 0, nullptr, nullptr, nullptr, nullptr,
                        s->stream))
    return rc;
  CUDA_TRY(get_parts<double>({{Minv, R.Mi}, {Linv, R.L}}, d, n, ns, s->stream));
  return 0;
}

static int minv_jvp_check(tds_b200_sim* s, const void* q, int K, const int* links, const double* local, int m, const void* t_q,
                          const void* t_par, const void* Linv, const void* t_Minv, const void* t_Linv) {
  if (int rc = minv_check(s, q, K, links, local, t_Minv, t_Linv)) return rc;
  if (Linv && K < 1) { set_err("mass inverse: J M^-1 J^T needs K >= 1 points"); return -1; }
  if (m < 1 || (!t_q && !t_par)) return -1;
  return par_without_installed(s, t_par, "mass inverse jvp: parameter tangents");
}

int tds_b200_mass_inverse_jvp_device(tds_b200_sim* s, const float* q, int K, const int* links, const double* local, int m, const double* t_q,
                                     const double* t_par, double* Minv, double* Linv, double* t_Minv, double* t_Linv, void* stream) {
  if (int rc = minv_jvp_check(s, q, K, links, local, m, t_q, t_par, Linv, t_Minv, t_Linv)) return rc;
  return minv_run(s, q, K, links, local, Minv, Linv, m, t_q, t_par, t_Minv, t_Linv, (cudaStream_t)stream);
}

int tds_b200_mass_inverse_jvp_host(tds_b200_sim* s, const double* q, int K, const int* links, const double* local, int m, const double* t_q,
                                   const double* t_par, double* Minv, double* Linv, double* t_Minv, double* t_Linv) {
  if (int rc = minv_jvp_check(s, q, K, links, local, m, t_q, t_par, Linv, t_Minv, t_Linv)) return rc;
  if (int rc = enter_derivative_host(s)) return rc;
  const int n = s->n, ns = s->ns;
  const MinvRows R = minv_rows(s, K);
  // tangents: host [n][dim][m] <-> device [dim * m][ns]; t_q | t_par | t_Minv | t_Linv | Minv | Linv
  const size_t tq = (size_t)(t_q ? s->dm[0].n_q : 0) * m, tp = (size_t)(t_par ? s->par.n : 0) * m, to = R.all() * m;
  if (int rc = put_q(s, q)) return rc;
  CUDA_TRY(grow_dev(&s->jac_dev, &s->jac_dev_bytes, sizeof(double) * (tq + tp + to + R.all() + 1) * ns));
  double* d = s->jac_dev;
  double* to_d = d + (tq + tp) * ns;
  double* v_d = to_d + to * ns;
  CUDA_TRY(put_parts<double>(d, {{t_q, tq}, {t_par, tp}}, n, ns, s->stream));
  if (int rc = minv_run(s, s->q, K, links, local, Minv ? v_d : nullptr, Linv ? v_d + R.Mi * ns : nullptr, m, t_q ? d : nullptr,
                        t_par ? d + tq * ns : nullptr, t_Minv ? to_d : nullptr, t_Linv ? to_d + R.Mi * m * ns : nullptr, s->stream))
    return rc;
  CUDA_TRY(get_parts<double>({{t_Minv, R.Mi * m}, {t_Linv, R.L * m}, {Minv, R.Mi}, {Linv, R.L}}, to_d, n, ns, s->stream));
  return 0;
}

static int minv_vjp_check(tds_b200_sim* s, const void* q, int K, const int* links, const double* local, const void* G_Minv,
                          const void* G_Linv, const void* g_q, const void* g_par) {
  if (int rc = minv_check(s, q, K, links, local, G_Minv, G_Linv)) return rc;
  if (!g_q && !g_par) return -1;
  return par_without_installed(s, g_par, "mass inverse vjp: parameter cotangents");
}

int tds_b200_mass_inverse_vjp_device(tds_b200_sim* s, const float* q, int K, const int* links, const double* local, const double* G_Minv,
                                     const double* G_Linv, double* g_q, double* g_par, void* stream) {
  if (int rc = minv_vjp_check(s, q, K, links, local, G_Minv, G_Linv, g_q, g_par)) return rc;
  const int n_q = s->dm[0].n_q, k = s->par.n;
  const MinvRows R = minv_rows(s, K);
  const size_t rows = R.Mi + (G_Linv ? R.L : 0);
  cudaStream_t sm = (cudaStream_t)stream;
  // the concatenated cotangent M^-1 (| Lambda^-1) (zero where a part is NULL), then g_q | g_par as one array for the contraction
  CUDA_TRY(grow_dev(&s->vjp_g, &s->vjp_g_bytes, sizeof(double) * (rows + n_q + k) * s->ns));
  double* g_d = s->vjp_g + rows * s->ns;
  CUDA_TRY(put_parts_d2d<double>(s->vjp_g, {{G_Minv, R.Mi}, {G_Linv, rows - R.Mi}}, s->ns, sm));
  if (int rc = minv_vjp_run(s, q, K, links, local, G_Linv != nullptr, s->vjp_g, g_q ? g_d : nullptr,
                            g_par ? g_d + (size_t)n_q * s->ns : nullptr, sm))
    return rc;
  CUDA_TRY(get_parts_d2d<double>({{g_q, (size_t)n_q}, {g_par, (size_t)k}}, g_d, s->ns, sm));
  return 0;
}

int tds_b200_mass_inverse_vjp_host(tds_b200_sim* s, const double* q, int K, const int* links, const double* local, const double* G_Minv,
                                   const double* G_Linv, double* g_q, double* g_par) {
  if (int rc = minv_vjp_check(s, q, K, links, local, G_Minv, G_Linv, g_q, g_par)) return rc;
  if (int rc = enter_derivative_host(s)) return rc;
  const int n = s->n, ns = s->ns, n_q = s->dm[0].n_q, k = s->par.n;
  const MinvRows R = minv_rows(s, K);
  const size_t rows = R.Mi + (G_Linv ? R.L : 0);
  if (int rc = put_q(s, q)) return rc;
  // G (M^-1 (| Lambda^-1), zero where a part is NULL) | g_q | g_par
  CUDA_TRY(grow_dev(&s->vjp_g, &s->vjp_g_bytes, sizeof(double) * (rows + n_q + k + 1) * ns));
  double* g_d = s->vjp_g + rows * ns;
  CUDA_TRY(put_parts<double>(s->vjp_g, {{G_Minv, R.Mi}, {G_Linv, rows - R.Mi}}, n, ns, s->stream));
  if (int rc = minv_vjp_run(s, s->q, K, links, local, G_Linv != nullptr, s->vjp_g, g_q ? g_d : nullptr,
                            g_par ? g_d + (size_t)n_q * ns : nullptr, s->stream))
    return rc;
  CUDA_TRY(get_parts<double>({{g_q, (size_t)n_q}, {g_par, (size_t)k}}, g_d, n, ns, s->stream));
  return 0;
}

// ---- point-constrained forward dynamics (DESIGN.md section 7.21): h = ID(q, qd, 0), M^-1, the point Jacobian and its drift from the INV,
// MINV and MOT instances of the world-frame kernel (inv_run, the mass inverse's value launch, mot_run, and their JVPs through
// jacobian_run), then the rows and the solve of tds_constrained.cu.  The inputs q | qd | tau are those of inverse dynamics with tau in the
// qdd slot (inv_n_in, put_inv_inputs).
struct CdynCall { int K; const int* links; const double* local; int dims; double eps; };

// tangents [j0, j0 + mc) of src [rows * m][ns] -> dst [rows * mc][ns] (src NULL: zeros)
static cudaError_t tangent_slice(double* dst, const double* src, size_t rows, int m, int j0, int mc, size_t ns, cudaStream_t sm) {
  if (!rows) return cudaSuccess;
  if (!src) return cudaMemsetAsync(dst, 0, sizeof(double) * rows * mc * ns, sm);
  return cudaMemcpy2DAsync(dst, sizeof(double) * mc * ns, src + (size_t)j0 * ns, sizeof(double) * m * ns, sizeof(double) * mc * ns, rows,
                           cudaMemcpyDeviceToDevice, sm);
}

static int cdyn_launch(tds_b200_sim* s, const TdsCdynCall& c, bool dual, cudaStream_t sm) {
  const int rc = tds_launch_cdyn(&c, dual ? 1 : 0, s->n, s->ns, sm);
  if (rc) set_err(std::string("constrained dynamics launch: ") + cudaGetErrorString((cudaError_t)rc));
  return rc;
}

// h = ID(q, qd, 0) [n_qd][ns] and M^-1 [n_qd^2][ns] from q [n_q][ns] and qd [n_qd][ns] fp32 (NULL: zero) by the INV and MINV value
// launches: what the constrained dynamics and the forward dynamics' derivatives start from (`what` names the call in errors)
static int h_minv_run(tds_b200_sim* s, const char* what, const float* q, const float* qd, double* h, double* Mi, cudaStream_t sm) {
  if (int rc = inv_run(s, q, qd, nullptr, h, sm)) return rc;
  return value_run(s, what, q, nullptr, nullptr, Mi, [&](const StepIO* io, const ParMap* pm) {
    return tds_launch_mass_inverse(&s->dm_m, io, pm, s->jac_scratch, sm);
  });
}

// The tangents of directions [j0, j0 + mc) of m that the constrained dynamics and the forward dynamics' derivatives share, laid out from
// w: T = the q | qd | 0 tangents [(n_q + 2 n_qd) * mc][ns] of the INV (and MOT) JVPs, Tp = t_par [k * mc], Tt = t_tau [n_qd * mc], and
// dh [n_qd * mc] and dM^-1 [n_qd^2 * mc] by the INV and MINV JVPs where the tangents given reach them (d_h, d_Mi).  `end` is where the
// caller's own tangents of the chunk begin; chunk_tangent_words(s) words per direction come before it.
struct ChunkTangents { double *T, *Tp, *Tt, *dh, *dMi, *end; bool d_h, d_Mi; };
static size_t chunk_tangent_words(const tds_b200_sim* s) {
  const size_t nd = s->dm[0].n_qd;
  return (size_t)inv_n_in(s) + s->par.n + 2 * nd + nd * nd;
}
static int chunk_tangents(tds_b200_sim* s, const float* q, const float* qd, int m, int j0, int mc, const double* t_q, const double* t_qd,
                          const double* t_tau, const double* t_par, double* w, ChunkTangents* c, cudaStream_t sm) {
  const int nd = s->dm[0].n_qd, n_q = s->dm[0].n_q, k = s->par.n;
  const size_t ns = s->ns, nn = (size_t)nd * nd, n_in = (size_t)inv_n_in(s);
  c->T = w;
  c->Tp = c->T + n_in * mc * ns;
  c->Tt = c->Tp + (size_t)k * mc * ns;
  c->dh = c->Tt + (size_t)nd * mc * ns;
  c->dMi = c->dh + (size_t)nd * mc * ns;
  c->end = c->dMi + nn * mc * ns;
  c->d_h = t_q || t_qd || t_par;
  c->d_Mi = t_q || t_par;
  CUDA_TRY(tangent_slice(c->T, t_q, n_q, m, j0, mc, ns, sm));
  CUDA_TRY(tangent_slice(c->T + (size_t)n_q * mc * ns, t_qd, nd, m, j0, mc, ns, sm));
  CUDA_TRY(tangent_slice(c->T + (size_t)(n_q + nd) * mc * ns, nullptr, nd, m, j0, mc, ns, sm));
  if (t_par) CUDA_TRY(tangent_slice(c->Tp, t_par, k, m, j0, mc, ns, sm));
  if (t_tau) CUDA_TRY(tangent_slice(c->Tt, t_tau, nd, m, j0, mc, ns, sm));
  if (c->d_h) {
    const JvpTangents jv{c->T, t_par ? c->Tp : nullptr, mc, Query::inv};
    if (int rc = jacobian_run(s, TDS_B200_MODE_FULL, 0, q, qd, nullptr, c->dh, sm, false, &jv)) return rc;
  }
  if (c->d_Mi) {   // (the qd tangents do not enter M^-1)
    const JvpTangents jv{t_q ? c->T : nullptr, t_par ? c->Tp : nullptr, mc, Query::minv};
    if (int rc = jacobian_run(s, TDS_B200_MODE_FULL, 0, q, nullptr, nullptr, c->dMi, sm, false, &jv)) return rc;
  }
  return 0;
}

// qdd [n_qd][ns] and f [R][ns] (R = dims K; either may be NULL) from q [n_q][ns], qd and tau [n_qd][ns] fp32 (either NULL: zero) and,
// with m >= 1 tangents t_q [n_q * m][ns], t_qd and t_tau [n_qd * m][ns], t_par [k * m][ns] (each may be NULL: zero), their tangents
// t_qdd [n_qd * m][ns] and t_f [R * m][ns] (either may be NULL).  Everything else goes to s->cdyn_dev: the values of h, M^-1, J, the
// drift and the value solve's scratch, then the tangents of one chunk of directions (within 1 GB) after another.
static int cdyn_run(tds_b200_sim* s, const float* q, const float* qd, const float* tau, const CdynCall& cc, double* qdd, double* f, int m,
                    const double* t_q, const double* t_qd, const double* t_tau, const double* t_par, double* t_qdd, double* t_f,
                    cudaStream_t sm) {
  const DevModel& D = s->dm[0];
  const int K = cc.K, nd = D.n_qd;
  const size_t ns = s->ns, nn = (size_t)nd * nd, nJ = (size_t)6 * K * nd, nA = (size_t)6 * K, R = (size_t)cc.dims * K;
  const size_t scr = R * nd + R * R + R;
  const bool tan = m > 0 && (t_qdd || t_f);
  // per tangent of a chunk: the shared tangents (chunk_tangents), dJ, d drift, and the (value, tangent) pairs of the scratch
  const size_t per = chunk_tangent_words(s) + nJ + nA + 2 * scr;
  const size_t fit = std::max<size_t>(1, ((size_t)1 << 30) / (sizeof(double) * per * ns));
  const int chunk = tan ? (int)std::min<size_t>(std::min<size_t>((size_t)m, 65535), fit) : 0;   // (gridDim.y, gridDim.z)
  CUDA_TRY(grow_dev(&s->cdyn_dev, &s->cdyn_dev_bytes, sizeof(double) * (nd + nn + nJ + nA + scr + per * chunk + 1) * ns));
  double* const h = s->cdyn_dev;
  double* const Mi = h + nd * ns;
  double* const J = Mi + nn * ns;
  double* const acc = J + nJ * ns;
  double* const Y = acc + nA * ns;
  double* const w = Y + scr * ns;
  if (int rc = h_minv_run(s, "constrained dynamics", q, qd, h, Mi, sm)) return rc;
  if (K > 0) {
    const TdsMotCall mc{K, cc.links, cc.local, J, nullptr, acc};
    if (int rc = mot_run(s, q, qd, nullptr, &mc, sm)) return rc;
  }
  TdsCdynCall c;
  memset(&c, 0, sizeof(c));
  c.K = K; c.dims = cc.dims; c.n_qd = nd; c.m = 1; c.m_out = 1; c.eps = cc.eps;
  c.tau = tau; c.h = h; c.Mi = Mi; c.J = J; c.acc = acc;
  c.Y = Y; c.A = Y + R * nd * ns; c.b = c.A + R * R * ns;
  if (qdd || f) {
    c.qdd = qdd; c.f = f;
    if (int rc = cdyn_launch(s, c, false, sm)) return rc;
  }
  if (!tan) return 0;
  const bool d_J = K > 0 && (t_q || t_qd);
  for (int j0 = 0; j0 < m; j0 += chunk) {
    const int mc = std::min(chunk, m - j0);
    ChunkTangents ct;
    if (int rc = chunk_tangents(s, q, qd, m, j0, mc, t_q, t_qd, t_tau, t_par, w, &ct, sm)) return rc;
    double* const dJ = ct.end;
    double* const dacc = dJ + nJ * mc * ns;
    double* const P = dacc + nA * mc * ns;   // Y | dY | A | dA | b | db
    if (d_J) {
      const TdsMotCall dmc{K, cc.links, cc.local, dJ, nullptr, dacc};
      if (int rc = mot_jvp_run(s, q, qd, nullptr, &dmc, mc, ct.T, sm)) return rc;
    }
    TdsCdynCall dc = c;
    dc.m = mc; dc.j0 = j0; dc.m_out = m;
    dc.dtau = t_tau ? ct.Tt : nullptr; dc.dh = ct.d_h ? ct.dh : nullptr; dc.dMi = ct.d_Mi ? ct.dMi : nullptr;
    dc.dJ = d_J ? dJ : nullptr; dc.dacc = d_J ? dacc : nullptr;
    dc.Y = P; dc.dY = dc.Y + R * nd * mc * ns; dc.A = dc.dY + R * nd * mc * ns; dc.dA = dc.A + R * R * mc * ns;
    dc.b = dc.dA + R * R * mc * ns; dc.db = dc.b + R * mc * ns;
    dc.qdd = t_qdd; dc.f = t_f;
    if (int rc = cdyn_launch(s, dc, true, sm)) return rc;
  }
  return 0;
}

// g_in [n_q + 2 n_qd][ns] (q | qd | tau, contiguous) and g_par [k][ns] (NULL: not wanted) = <G, d(qdd | f)>, G [n_qd + R][ns]
static int cdyn_vjp_run(tds_b200_sim* s, const float* q, const float* qd, const float* tau, const CdynCall& cc, const double* G,
                        double* g_in, double* g_par, cudaStream_t sm) {
  const size_t ns = s->ns, n_q = s->dm[0].n_q, nd = s->dm[0].n_qd, R = (size_t)cc.dims * cc.K;
  return vjp_by_eye(s, "constrained dynamics", inv_n_in(s), nd + R, G, g_in, g_par, sm,
                    [&](int m, const double* t_in, const double* t_par, double* dO) {
                      return cdyn_run(s, q, qd, tau, cc, nullptr, nullptr, m, t_in, t_in + n_q * m * ns, t_in + (n_q + nd) * m * ns, t_par,
                                      dO, R ? dO + nd * m * ns : nullptr, sm);
                    });
}

// -1: no q, no output (tangent output, cotangent), K out of [0, TDS_B200_MAX_OSIM_POINTS], dims not 3 or 6, damping negative or not
// finite, f (t_f, G_f) with K = 0, a missing or bad point table
static int cdyn_check(tds_b200_sim* s, const void* q, const CdynCall& cc, const void* qdd, const void* f) {
  if (!s || !q || (!qdd && !f)) return -1;
  if (cc.K < 0 || cc.K > TDS_B200_MAX_OSIM_POINTS) { set_err("constrained dynamics: K out of [0, TDS_B200_MAX_OSIM_POINTS]"); return -1; }
  if (cc.dims != 3 && cc.dims != 6) { set_err("constrained dynamics: dims is 3 or 6"); return -1; }
  if (!(cc.eps >= 0.0) || !std::isfinite(cc.eps)) { set_err("constrained dynamics: damping must be finite and >= 0"); return -1; }
  if (f && cc.K < 1) { set_err("constrained dynamics: f needs K >= 1 points"); return -1; }
  return kin_check(s, q, cc.K, cc.links, cc.local);
}

int tds_b200_constrained_dynamics_device(tds_b200_sim* s, const float* q, const float* qd, const float* tau, int K, const int* links,
                                         const double* local, int dims, double damping, double* qdd, double* f, void* stream) {
  const CdynCall cc{K, links, local, dims, damping};
  if (int rc = cdyn_check(s, q, cc, qdd, f)) return rc;
  return cdyn_run(s, q, qd, tau, cc, qdd, f, 0, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, (cudaStream_t)stream);
}

int tds_b200_constrained_dynamics_host(tds_b200_sim* s, const double* q, const double* qd, const double* tau, int K, const int* links,
                                       const double* local, int dims, double damping, double* qdd, double* f) {
  const CdynCall cc{K, links, local, dims, damping};
  if (int rc = cdyn_check(s, q, cc, qdd, f)) return rc;
  if (int rc = enter_derivative_host(s)) return rc;
  const int n = s->n, ns = s->ns;
  const size_t nd = s->dm[0].n_qd, R = (size_t)dims * K;
  const float *qd_d, *tau_d;
  if (int rc = put_inv_inputs(s, q, qd, tau, &qd_d, &tau_d)) return rc;
  CUDA_TRY(grow_dev(&s->jac_dev, &s->jac_dev_bytes, sizeof(double) * (nd + R + 1) * ns));
  double* d = s->jac_dev;
  if (int rc = cdyn_run(s, s->q, qd_d, tau_d, cc, qdd ? d : nullptr, f ? d + nd * ns : nullptr, 0, nullptr, nullptr, nullptr, nullptr, nullptr,
                        nullptr, s->stream))
    return rc;
  CUDA_TRY(get_parts<double>({{qdd, nd}, {f, R}}, d, n, ns, s->stream));
  return 0;
}

static int cdyn_jvp_check(tds_b200_sim* s, const void* q, const CdynCall& cc, int m, const void* t_q, const void* t_qd, const void* t_tau,
                          const void* t_par, const void* f, const void* t_qdd, const void* t_f) {
  if (int rc = cdyn_check(s, q, cc, t_qdd, t_f)) return rc;
  if (f && cc.K < 1) { set_err("constrained dynamics: f needs K >= 1 points"); return -1; }
  if (m < 1 || (!t_q && !t_qd && !t_tau && !t_par)) return -1;
  return par_without_installed(s, t_par, "constrained dynamics jvp: parameter tangents");
}

int tds_b200_constrained_dynamics_jvp_device(tds_b200_sim* s, const float* q, const float* qd, const float* tau, int K, const int* links,
                                             const double* local, int dims, double damping, int m, const double* t_q, const double* t_qd,
                                             const double* t_tau, const double* t_par, double* qdd, double* f, double* t_qdd, double* t_f,
                                             void* stream) {
  const CdynCall cc{K, links, local, dims, damping};
  if (int rc = cdyn_jvp_check(s, q, cc, m, t_q, t_qd, t_tau, t_par, f, t_qdd, t_f)) return rc;
  return cdyn_run(s, q, qd, tau, cc, qdd, f, m, t_q, t_qd, t_tau, t_par, t_qdd, t_f, (cudaStream_t)stream);
}

int tds_b200_constrained_dynamics_jvp_host(tds_b200_sim* s, const double* q, const double* qd, const double* tau, int K, const int* links,
                                           const double* local, int dims, double damping, int m, const double* t_q, const double* t_qd,
                                           const double* t_tau, const double* t_par, double* qdd, double* f, double* t_qdd, double* t_f) {
  const CdynCall cc{K, links, local, dims, damping};
  if (int rc = cdyn_jvp_check(s, q, cc, m, t_q, t_qd, t_tau, t_par, f, t_qdd, t_f)) return rc;
  if (int rc = enter_derivative_host(s)) return rc;
  const int n = s->n, ns = s->ns;
  const size_t n_q = s->dm[0].n_q, nd = s->dm[0].n_qd, R = (size_t)dims * K;
  // tangents: host [n][dim][m] <-> device [dim * m][ns]; t_q | t_qd | t_tau | t_par | t_qdd | t_f | qdd | f
  const size_t tq = (t_q ? n_q : 0) * m, tqd = (t_qd ? nd : 0) * m, tt = (t_tau ? nd : 0) * m, tp = (size_t)(t_par ? s->par.n : 0) * m;
  const size_t ti = tq + tqd + tt + tp, to = (nd + R) * m;
  const float *qd_d, *tau_d;
  if (int rc = put_inv_inputs(s, q, qd, tau, &qd_d, &tau_d)) return rc;
  CUDA_TRY(grow_dev(&s->jac_dev, &s->jac_dev_bytes, sizeof(double) * (ti + to + nd + R + 1) * ns));
  double* d = s->jac_dev;
  double* to_d = d + ti * ns;
  double* v_d = to_d + to * ns;
  CUDA_TRY(put_parts<double>(d, {{t_q, tq}, {t_qd, tqd}, {t_tau, tt}, {t_par, tp}}, n, ns, s->stream));
  if (int rc = cdyn_run(s, s->q, qd_d, tau_d, cc, qdd ? v_d : nullptr, f ? v_d + nd * ns : nullptr, m, t_q ? d : nullptr,
                        t_qd ? d + tq * ns : nullptr, t_tau ? d + (tq + tqd) * ns : nullptr, t_par ? d + (tq + tqd + tt) * ns : nullptr,
                        t_qdd ? to_d : nullptr, t_f ? to_d + nd * m * ns : nullptr, s->stream))
    return rc;
  CUDA_TRY(get_parts<double>({{t_qdd, nd * m}, {t_f, R * m}, {qdd, nd}, {f, R}}, to_d, n, ns, s->stream));
  return 0;
}

static int cdyn_vjp_check(tds_b200_sim* s, const void* q, const CdynCall& cc, const void* G_qdd, const void* G_f, const void* g_q,
                          const void* g_qd, const void* g_tau, const void* g_par) {
  if (int rc = cdyn_check(s, q, cc, G_qdd, G_f)) return rc;
  if (!g_q && !g_qd && !g_tau && !g_par) return -1;
  return par_without_installed(s, g_par, "constrained dynamics vjp: parameter cotangents");
}

int tds_b200_constrained_dynamics_vjp_device(tds_b200_sim* s, const float* q, const float* qd, const float* tau, int K, const int* links,
                                             const double* local, int dims, double damping, const double* G_qdd, const double* G_f,
                                             double* g_q, double* g_qd, double* g_tau, double* g_par, void* stream) {
  const CdynCall cc{K, links, local, dims, damping};
  if (int rc = cdyn_vjp_check(s, q, cc, G_qdd, G_f, g_q, g_qd, g_tau, g_par)) return rc;
  const size_t n_q = s->dm[0].n_q, nd = s->dm[0].n_qd, R = (size_t)dims * K, k = s->par.n, n_in = inv_n_in(s);
  cudaStream_t sm = (cudaStream_t)stream;
  // the concatenated cotangent qdd | f (zero where a part is NULL), then g_q | g_qd | g_tau | g_par as one array for the contraction
  CUDA_TRY(grow_dev(&s->vjp_g, &s->vjp_g_bytes, sizeof(double) * (nd + R + n_in + k) * s->ns));
  double* g_d = s->vjp_g + (nd + R) * s->ns;
  CUDA_TRY(put_parts_d2d<double>(s->vjp_g, {{G_qdd, nd}, {G_f, R}}, s->ns, sm));
  if (int rc = cdyn_vjp_run(s, q, qd, tau, cc, s->vjp_g, g_d, g_par ? g_d + n_in * s->ns : nullptr, sm)) return rc;
  CUDA_TRY(get_parts_d2d<double>({{g_q, n_q}, {g_qd, nd}, {g_tau, nd}, {g_par, g_par ? k : 0}}, g_d, s->ns, sm));
  return 0;
}

int tds_b200_constrained_dynamics_vjp_host(tds_b200_sim* s, const double* q, const double* qd, const double* tau, int K, const int* links,
                                           const double* local, int dims, double damping, const double* G_qdd, const double* G_f,
                                           double* g_q, double* g_qd, double* g_tau, double* g_par) {
  const CdynCall cc{K, links, local, dims, damping};
  if (int rc = cdyn_vjp_check(s, q, cc, G_qdd, G_f, g_q, g_qd, g_tau, g_par)) return rc;
  if (int rc = enter_derivative_host(s)) return rc;
  const int n = s->n, ns = s->ns;
  const size_t n_q = s->dm[0].n_q, nd = s->dm[0].n_qd, R = (size_t)dims * K, k = s->par.n, n_in = inv_n_in(s);
  const float *qd_d, *tau_d;
  if (int rc = put_inv_inputs(s, q, qd, tau, &qd_d, &tau_d)) return rc;
  // G (qdd | f, zero where a part is NULL) | g_q | g_qd | g_tau | g_par
  CUDA_TRY(grow_dev(&s->vjp_g, &s->vjp_g_bytes, sizeof(double) * (nd + R + n_in + k + 1) * ns));
  double* g_d = s->vjp_g + (nd + R) * ns;
  CUDA_TRY(put_parts<double>(s->vjp_g, {{G_qdd, nd}, {G_f, R}}, n, ns, s->stream));
  if (int rc = cdyn_vjp_run(s, s->q, qd_d, tau_d, cc, s->vjp_g, g_d, g_par ? g_d + n_in * ns : nullptr, s->stream)) return rc;
  CUDA_TRY(get_parts<double>({{g_q, n_q}, {g_qd, nd}, {g_tau, nd}, {g_par, g_par ? k : 0}}, g_d, n, ns, s->stream));
  return 0;
}

// ---- derivatives of the forward dynamics d qdd / dq, d qdd / dqd, d qdd / dtau (DESIGN.md section 7.24): h and M^-1 from the INV and
// MINV instances and qdd from the constrained dynamics' solve at K = 0 (the launches of cdyn_run), d tau / dq and d tau / dqd from the DER
// instances at that fp64 qdd (der_run, der_jvp_run), then the product kernel of tds_fd_derivatives.cu.  The inputs q | qd | tau are those
// of the constrained dynamics (inv_n_in, put_inv_inputs).
// The four outputs qdd [n_qd][ns], d qdd / dq, d qdd / dqd and d qdd / dtau [n_qd * n_qd][ns] (each may be NULL), or their tangents
// [rows * m][ns]
struct FddOut { double* qdd; double* dq; double* dqd; double* dtau; };

static int fdd_launch(tds_b200_sim* s, const TdsFddCall& c, bool dual, cudaStream_t sm) {
  const int rc = tds_launch_fdd(&c, dual ? 1 : 0, s->n, s->ns, sm);
  if (rc) set_err(std::string("forward dynamics derivatives launch: ") + cudaGetErrorString((cudaError_t)rc));
  return rc;
}

// The outputs o from q [n_q][ns], qd and tau [n_qd][ns] fp32 (either NULL: zero) and, with m >= 1 tangents t_q [n_q * m][ns], t_qd and
// t_tau [n_qd * m][ns], t_par [k * m][ns] (each may be NULL: zero), their tangents t.  Everything else goes to s->cdyn_dev: the values of
// h, M^-1 (unless o.dtau takes it), qdd (unless o.qdd takes it), d tau / dq and d tau / dqd, then the tangents of one chunk of directions
// (within 1 GB) after another.  dM^-1 of a chunk serves both the solve and the product.
static int fdd_run(tds_b200_sim* s, const float* q, const float* qd, const float* tau, const FddOut& o, int m, const double* t_q,
                   const double* t_qd, const double* t_tau, const double* t_par, const FddOut& t, cudaStream_t sm) {
  const DevModel& D = s->dm[0];
  const int nd = D.n_qd, n_q = D.n_q;
  const size_t ns = s->ns, nn = (size_t)nd * nd;
  const bool tan = m > 0 && (t.qdd || t.dq || t.dqd || t.dtau), tan_A = tan && (t.dq || t.dqd);
  const bool want_A = o.dq || o.dqd || tan_A;
  // per tangent of a chunk: the shared tangents (chunk_tangents), d(d tau / dq), d(d tau / dqd)
  const size_t per = chunk_tangent_words(s) + 2 * nn;
  const size_t fit = std::max<size_t>(1, ((size_t)1 << 30) / (sizeof(double) * per * ns));
  const int chunk = tan ? (int)std::min<size_t>(std::min<size_t>((size_t)m, 65535), fit) : 0;   // (gridDim.z)
  CUDA_TRY(grow_dev(&s->cdyn_dev, &s->cdyn_dev_bytes, sizeof(double) * (3 * (size_t)nd + 3 * nn + per * chunk + 1) * ns));
  double* const h = s->cdyn_dev;
  double* const Mi = o.dtau ? o.dtau : h + nd * ns;
  double* const qdd = o.qdd ? o.qdd : h + (nd + nn) * ns;
  double* const Aq = h + (2 * nd + nn) * ns;
  double* const Aqd = Aq + nn * ns;
  double* const w = Aqd + nn * ns;
  if (int rc = h_minv_run(s, "forward dynamics derivatives", q, qd, h, Mi, sm)) return rc;
  TdsCdynCall c;   // the constrained dynamics' solve without points: qdd = M^-1 (tau - h)
  memset(&c, 0, sizeof(c));
  c.dims = 3; c.n_qd = nd; c.m = 1; c.m_out = 1;
  c.tau = tau; c.h = h; c.Mi = Mi; c.qdd = qdd;
  if (int rc = cdyn_launch(s, c, false, sm)) return rc;
  if (want_A) { if (int rc = der_run(s, q, qd, nullptr, Aq, Aqd, sm, qdd)) return rc; }
  TdsFddCall pc;
  memset(&pc, 0, sizeof(pc));
  pc.n_qd = nd; pc.m = 1; pc.m_out = 1; pc.Mi = Mi; pc.Aq = Aq; pc.Aqd = Aqd;
  if (o.dq || o.dqd) {
    pc.dq = o.dq; pc.dqd = o.dqd;
    if (int rc = fdd_launch(s, pc, false, sm)) return rc;
  }
  if (!tan) return 0;
  for (int j0 = 0; j0 < m; j0 += chunk) {
    const int mc = std::min(chunk, m - j0);
    ChunkTangents ct;
    if (int rc = chunk_tangents(s, q, qd, m, j0, mc, t_q, t_qd, t_tau, t_par, w, &ct, sm)) return rc;
    double* const Tqdd = ct.T + (size_t)(n_q + nd) * mc * ns;   // the qdd tangents: zero for the INV JVP, then the solve's dqdd
    double* const dAq = ct.end;
    double* const dAqd = dAq + nn * mc * ns;
    TdsCdynCall dc = c;   // dqdd into the qdd tangents of the DER JVP
    dc.m = mc; dc.j0 = 0; dc.m_out = mc;
    dc.dtau = t_tau ? ct.Tt : nullptr; dc.dh = ct.d_h ? ct.dh : nullptr; dc.dMi = ct.d_Mi ? ct.dMi : nullptr;
    dc.qdd = Tqdd;
    if (int rc = cdyn_launch(s, dc, true, sm)) return rc;
    if (t.qdd)
      CUDA_TRY(cudaMemcpy2DAsync(t.qdd + (size_t)j0 * ns, sizeof(double) * m * ns, Tqdd, sizeof(double) * mc * ns, sizeof(double) * mc * ns,
                                 nd, cudaMemcpyDeviceToDevice, sm));
    if (tan_A) {
      if (int rc = der_jvp_run(s, q, qd, nullptr, mc, ct.T, t_par ? ct.Tp : nullptr, nullptr, nullptr, t.dq ? dAq : nullptr,
                               t.dqd ? dAqd : nullptr, sm, qdd))
        return rc;
    }
    if (!tan_A && !t.dtau) continue;
    TdsFddCall dp = pc;
    dp.m = mc; dp.j0 = j0; dp.m_out = m;
    dp.dMi = ct.d_Mi ? ct.dMi : nullptr; dp.dAq = dAq; dp.dAqd = dAqd;
    dp.dq = t.dq; dp.dqd = t.dqd; dp.dtau = t.dtau;
    if (int rc = fdd_launch(s, dp, true, sm)) return rc;
  }
  return 0;
}

// g_in [n_q + 2 n_qd][ns] (q | qd | tau, contiguous) and g_par [k][ns] (NULL: not wanted) = <G, d(qdd | d qdd / dq | d qdd / dqd |
// d qdd / dtau)>, G [n_qd + 3 n_qd^2][ns]
static int fdd_vjp_run(tds_b200_sim* s, const float* q, const float* qd, const float* tau, const double* G, double* g_in, double* g_par,
                       cudaStream_t sm) {
  const size_t ns = s->ns, n_q = s->dm[0].n_q, nd = s->dm[0].n_qd, nn = nd * nd;
  return vjp_by_eye(s, "forward dynamics derivatives", inv_n_in(s), nd + 3 * nn, G, g_in, g_par, sm,
                    [&](int m, const double* t_in, const double* t_par, double* dO) {
                      const size_t r = (size_t)m * ns;
                      const FddOut t{dO, dO + nd * r, dO + (nd + nn) * r, dO + (nd + 2 * nn) * r};
                      return fdd_run(s, q, qd, tau, FddOut{}, m, t_in, t_in + n_q * r, t_in + (n_q + nd) * r, t_par, t, sm);
                    });
}

static bool fdd_any(const void* a, const void* b, const void* c, const void* d) { return a || b || c || d; }

int tds_b200_forward_dynamics_derivatives_device(tds_b200_sim* s, const float* q, const float* qd, const float* tau, double* qdd,
                                                 double* dqdd_dq, double* dqdd_dqd, double* dqdd_dtau, void* stream) {
  if (!s || !q || !fdd_any(qdd, dqdd_dq, dqdd_dqd, dqdd_dtau)) return -1;
  return fdd_run(s, q, qd, tau, FddOut{qdd, dqdd_dq, dqdd_dqd, dqdd_dtau}, 0, nullptr, nullptr, nullptr, nullptr, FddOut{},
                 (cudaStream_t)stream);
}

int tds_b200_forward_dynamics_derivatives_host(tds_b200_sim* s, const double* q, const double* qd, const double* tau, double* qdd,
                                               double* dqdd_dq, double* dqdd_dqd, double* dqdd_dtau) {
  if (!s || !q || !fdd_any(qdd, dqdd_dq, dqdd_dqd, dqdd_dtau)) return -1;
  if (int rc = enter_derivative_host(s)) return rc;
  const int n = s->n, ns = s->ns;
  const size_t nd = s->dm[0].n_qd, nn = nd * nd;
  const float *qd_d, *tau_d;
  if (int rc = put_inv_inputs(s, q, qd, tau, &qd_d, &tau_d)) return rc;
  CUDA_TRY(grow_dev(&s->jac_dev, &s->jac_dev_bytes, sizeof(double) * (nd + 3 * nn + 1) * ns));
  double* d = s->jac_dev;
  const FddOut o{qdd ? d : nullptr, dqdd_dq ? d + nd * ns : nullptr, dqdd_dqd ? d + (nd + nn) * ns : nullptr,
                 dqdd_dtau ? d + (nd + 2 * nn) * ns : nullptr};
  if (int rc = fdd_run(s, s->q, qd_d, tau_d, o, 0, nullptr, nullptr, nullptr, nullptr, FddOut{}, s->stream)) return rc;
  CUDA_TRY(get_parts<double>({{qdd, nd}, {dqdd_dq, nn}, {dqdd_dqd, nn}, {dqdd_dtau, nn}}, d, n, ns, s->stream));
  return 0;
}

static int fdd_jvp_check(tds_b200_sim* s, const void* q, int m, const void* t_q, const void* t_qd, const void* t_tau, const void* t_par,
                         const FddOut& t) {
  if (!s || !q || !fdd_any(t.qdd, t.dq, t.dqd, t.dtau) || m < 1 || !fdd_any(t_q, t_qd, t_tau, t_par)) return -1;
  return par_without_installed(s, t_par, "forward dynamics derivatives jvp: parameter tangents");
}

int tds_b200_forward_dynamics_derivatives_jvp_device(tds_b200_sim* s, const float* q, const float* qd, const float* tau, int m,
                                                     const double* t_q, const double* t_qd, const double* t_tau, const double* t_par,
                                                     double* qdd, double* dqdd_dq, double* dqdd_dqd, double* dqdd_dtau, double* t_qdd,
                                                     double* t_dqdd_dq, double* t_dqdd_dqd, double* t_dqdd_dtau, void* stream) {
  const FddOut t{t_qdd, t_dqdd_dq, t_dqdd_dqd, t_dqdd_dtau};
  if (int rc = fdd_jvp_check(s, q, m, t_q, t_qd, t_tau, t_par, t)) return rc;
  return fdd_run(s, q, qd, tau, FddOut{qdd, dqdd_dq, dqdd_dqd, dqdd_dtau}, m, t_q, t_qd, t_tau, t_par, t, (cudaStream_t)stream);
}

int tds_b200_forward_dynamics_derivatives_jvp_host(tds_b200_sim* s, const double* q, const double* qd, const double* tau, int m,
                                                   const double* t_q, const double* t_qd, const double* t_tau, const double* t_par,
                                                   double* qdd, double* dqdd_dq, double* dqdd_dqd, double* dqdd_dtau, double* t_qdd,
                                                   double* t_dqdd_dq, double* t_dqdd_dqd, double* t_dqdd_dtau) {
  if (int rc = fdd_jvp_check(s, q, m, t_q, t_qd, t_tau, t_par, FddOut{t_qdd, t_dqdd_dq, t_dqdd_dqd, t_dqdd_dtau})) return rc;
  if (int rc = enter_derivative_host(s)) return rc;
  const int n = s->n, ns = s->ns;
  const size_t n_q = s->dm[0].n_q, nd = s->dm[0].n_qd, nn = nd * nd;
  // tangents: host [n][dim][m] <-> device [dim * m][ns]; t_q | t_qd | t_tau | t_par | the four output tangents | the four values
  const size_t tq = (t_q ? n_q : 0) * m, tqd = (t_qd ? nd : 0) * m, tt = (t_tau ? nd : 0) * m, tp = (size_t)(t_par ? s->par.n : 0) * m;
  const size_t ti = tq + tqd + tt + tp, to = (nd + 3 * nn) * m;
  const float *qd_d, *tau_d;
  if (int rc = put_inv_inputs(s, q, qd, tau, &qd_d, &tau_d)) return rc;
  CUDA_TRY(grow_dev(&s->jac_dev, &s->jac_dev_bytes, sizeof(double) * (ti + to + nd + 3 * nn + 1) * ns));
  double* d = s->jac_dev;
  double* to_d = d + ti * ns;
  double* v_d = to_d + to * ns;
  CUDA_TRY(put_parts<double>(d, {{t_q, tq}, {t_qd, tqd}, {t_tau, tt}, {t_par, tp}}, n, ns, s->stream));
  const size_t r = (size_t)m * ns;
  const FddOut o{qdd ? v_d : nullptr, dqdd_dq ? v_d + nd * ns : nullptr, dqdd_dqd ? v_d + (nd + nn) * ns : nullptr,
                 dqdd_dtau ? v_d + (nd + 2 * nn) * ns : nullptr};
  const FddOut t{t_qdd ? to_d : nullptr, t_dqdd_dq ? to_d + nd * r : nullptr, t_dqdd_dqd ? to_d + (nd + nn) * r : nullptr,
                 t_dqdd_dtau ? to_d + (nd + 2 * nn) * r : nullptr};
  if (int rc = fdd_run(s, s->q, qd_d, tau_d, o, m, t_q ? d : nullptr, t_qd ? d + tq * ns : nullptr, t_tau ? d + (tq + tqd) * ns : nullptr,
                       t_par ? d + (tq + tqd + tt) * ns : nullptr, t, s->stream))
    return rc;
  CUDA_TRY(get_parts<double>({{t_qdd, nd * m}, {t_dqdd_dq, nn * m}, {t_dqdd_dqd, nn * m}, {t_dqdd_dtau, nn * m}, {qdd, nd}, {dqdd_dq, nn},
                              {dqdd_dqd, nn}, {dqdd_dtau, nn}},
                             to_d, n, ns, s->stream));
  return 0;
}

static int fdd_vjp_check(tds_b200_sim* s, const void* q, const void* G_qdd, const void* G_dq, const void* G_dqd, const void* G_dtau,
                         const void* g_q, const void* g_qd, const void* g_tau, const void* g_par) {
  if (!s || !q || !fdd_any(G_qdd, G_dq, G_dqd, G_dtau) || !fdd_any(g_q, g_qd, g_tau, g_par)) return -1;
  return par_without_installed(s, g_par, "forward dynamics derivatives vjp: parameter cotangents");
}

int tds_b200_forward_dynamics_derivatives_vjp_device(tds_b200_sim* s, const float* q, const float* qd, const float* tau, const double* G_qdd,
                                                     const double* G_dq, const double* G_dqd, const double* G_dtau, double* g_q, double* g_qd,
                                                     double* g_tau, double* g_par, void* stream) {
  if (int rc = fdd_vjp_check(s, q, G_qdd, G_dq, G_dqd, G_dtau, g_q, g_qd, g_tau, g_par)) return rc;
  const size_t n_q = s->dm[0].n_q, nd = s->dm[0].n_qd, nn = nd * nd, k = s->par.n, n_in = inv_n_in(s), rows = nd + 3 * nn;
  cudaStream_t sm = (cudaStream_t)stream;
  // the concatenated cotangent (zero where a part is NULL), then g_q | g_qd | g_tau | g_par as one array for the contraction
  CUDA_TRY(grow_dev(&s->vjp_g, &s->vjp_g_bytes, sizeof(double) * (rows + n_in + k) * s->ns));
  double* g_d = s->vjp_g + rows * s->ns;
  CUDA_TRY(put_parts_d2d<double>(s->vjp_g, {{G_qdd, nd}, {G_dq, nn}, {G_dqd, nn}, {G_dtau, nn}}, s->ns, sm));
  if (int rc = fdd_vjp_run(s, q, qd, tau, s->vjp_g, g_d, g_par ? g_d + n_in * s->ns : nullptr, sm)) return rc;
  CUDA_TRY(get_parts_d2d<double>({{g_q, n_q}, {g_qd, nd}, {g_tau, nd}, {g_par, g_par ? k : 0}}, g_d, s->ns, sm));
  return 0;
}

int tds_b200_forward_dynamics_derivatives_vjp_host(tds_b200_sim* s, const double* q, const double* qd, const double* tau, const double* G_qdd,
                                                   const double* G_dq, const double* G_dqd, const double* G_dtau, double* g_q, double* g_qd,
                                                   double* g_tau, double* g_par) {
  if (int rc = fdd_vjp_check(s, q, G_qdd, G_dq, G_dqd, G_dtau, g_q, g_qd, g_tau, g_par)) return rc;
  if (int rc = enter_derivative_host(s)) return rc;
  const int n = s->n, ns = s->ns;
  const size_t n_q = s->dm[0].n_q, nd = s->dm[0].n_qd, nn = nd * nd, k = s->par.n, n_in = inv_n_in(s), rows = nd + 3 * nn;
  const float *qd_d, *tau_d;
  if (int rc = put_inv_inputs(s, q, qd, tau, &qd_d, &tau_d)) return rc;
  // G (qdd | d qdd / dq | d qdd / dqd | d qdd / dtau, zero where a part is NULL) | g_q | g_qd | g_tau | g_par
  CUDA_TRY(grow_dev(&s->vjp_g, &s->vjp_g_bytes, sizeof(double) * (rows + n_in + k + 1) * ns));
  double* g_d = s->vjp_g + rows * ns;
  CUDA_TRY(put_parts<double>(s->vjp_g, {{G_qdd, nd}, {G_dq, nn}, {G_dqd, nn}, {G_dtau, nn}}, n, ns, s->stream));
  if (int rc = fdd_vjp_run(s, s->q, qd_d, tau_d, s->vjp_g, g_d, g_par ? g_d + n_in * ns : nullptr, s->stream)) return rc;
  CUDA_TRY(get_parts<double>({{g_q, n_q}, {g_qd, nd}, {g_tau, nd}, {g_par, g_par ? k : 0}}, g_d, n, ns, s->stream));
  return 0;
}

// ---- vector-Jacobian product: g_in = g_out^T d(q', qd' | qdd) / d(q | qd | tau or action (| kp, kd, max_force)) by the taping
// instance of the world-frame kernel (tds_tape.cuh), one lane per environment.  Environments run in chunks that keep arena +
// tape + adjoints inside 2 GB; a chunk whose tape overflowed is rerun with twice the capacity (the flag is read after every
// chunk, so the call synchronises its stream once per chunk).
static int vjp_check(tds_b200_sim* s, int mode, int use_pd, const void* q, const void* qd, const void* g_out, const void* g_req) {
  if (!s || !q || !qd || !g_out || !g_req) return -1;
  if (mode == 3) { set_err("vjp: modes FD, NOCONTACT, FULL"); return -2; }
  if (use_pd && s->E.n_act == 0) { set_err("use_pd without tds_b200_set_env"); return -3; }
  return 0;
}

// warps of environments one launch of the taping instance takes at the current tape capacity: arena + tape + adjoints within 2 GB
static size_t tape_warps(const tds_b200_sim* s) {
  const size_t arena_warp = (size_t)s->dm_ad.x_total * 32 * 4;
  const size_t lane_bytes = (size_t)s->tape_cap * (sizeof(tds::TapeNode) + sizeof(double));
  const size_t warps = ((size_t)2 << 30) / (arena_warp + 32 * lane_bytes);
  return warps < 1 ? 1 : warps;
}

// g_in (may be null while parameters are installed) and g_par [k][ns] (or null); every pointer is offset per chunk of environments
static int vjp_run(tds_b200_sim* s, int mode, int use_pd, const float* q, const float* qd, const float* tau_or_action,
                   const double* g_out, double* g_in, double* g_par, void* stream) {
  ParMap pmv = s->par;
  const ParMap* pm = s->par.n > 0 ? &pmv : nullptr;
  cudaStream_t sm = (cudaStream_t)stream;
  const size_t arena_warp = (size_t)s->dm_ad.x_total * 32 * 4;
  if (!s->vjp_flag) CUDA_TRY(cudaMalloc((void**)&s->vjp_flag, sizeof(int)));
  const int n = s->n, ns = s->ns;
  for (int e0 = 0; e0 < n;) {
    size_t warps = tape_warps(s);
    const size_t left = (size_t)(n - e0 + 31) / 32;
    if (warps > left) warps = left;
    const int chunk = (int)(warps * 32 < (size_t)(n - e0) ? warps * 32 : (size_t)(n - e0));
    const size_t tape_b = warps * 32 * s->tape_cap * sizeof(tds::TapeNode), adj_b = warps * 32 * s->tape_cap * sizeof(double);
    const size_t need = warps * arena_warp + tape_b + adj_b;
    if (need > s->vjp_buf_bytes) CUDA_TRY(cudaStreamSynchronize(sm));   // (earlier chunks still use the buffer)
    CUDA_TRY(grow_dev(&s->vjp_buf, &s->vjp_buf_bytes, need));
    StepIO io;
    memset(&io, 0, sizeof(io));
    io.q_in = q + e0; io.qd_in = qd + e0; io.tau_in = tau_or_action ? tau_or_action + e0 : nullptr;   // [dim][ns]: column offset
    io.n = chunk; io.n_stride = ns;
    io.g_out = g_out + e0; io.g_in = g_in ? g_in + e0 : nullptr;
    pmv.values = s->par_dev ? s->par_dev + e0 : nullptr; pmv.grad = g_par ? g_par + e0 : nullptr;
    io.tape = s->vjp_buf + warps * arena_warp;
    io.tape_adj = (double*)(s->vjp_buf + warps * arena_warp + tape_b);
    io.tape_cap = s->tape_cap; io.tape_overflow = s->vjp_flag;
    CUDA_TRY(cudaMemsetAsync(s->vjp_flag, 0, sizeof(int), sm));
    int rc = pm ? tds_launch_stepw_vjp_par(&s->dm_ad, &s->P, &s->E, &io, pm, mode, use_pd, s->vjp_buf, sm)
                : tds_launch_stepw_vjp(&s->dm_ad, &s->P, &s->E, &io, mode, use_pd, s->vjp_buf, sm);
    if (rc) { set_err(std::string("vjp launch: ") + cudaGetErrorString((cudaError_t)rc)); return rc; }
    int overflow = 0;
    CUDA_TRY(cudaMemcpyAsync(&overflow, s->vjp_flag, sizeof(int), cudaMemcpyDeviceToHost, sm));
    CUDA_TRY(cudaStreamSynchronize(sm));
    if (overflow) {
      if (s->tape_cap > (1 << 28)) { set_err("vjp: tape capacity exhausted"); return -4; }
      s->tape_cap *= 2;
      continue;
    }
    e0 += chunk;
  }
  return 0;
}

int tds_b200_step_vjp_device(tds_b200_sim* s, int mode, int use_pd, const float* q, const float* qd, const float* tau_or_action,
                             const double* g_out, double* g_in, void* stream) {
  if (int rc = vjp_check(s, mode, use_pd, q, qd, g_out, g_in)) return rc;
  return vjp_run(s, mode, use_pd, q, qd, tau_or_action, g_out, g_in, nullptr, stream);
}

int tds_b200_step_vjp_params_device(tds_b200_sim* s, int mode, int use_pd, const float* q, const float* qd,
                                    const float* tau_or_action, const double* g_out, double* g_in, double* g_par, void* stream) {
  if (int rc = vjp_check(s, mode, use_pd, q, qd, g_out, g_par)) return rc;
  if (s->par.n == 0) { set_err("parameter vjp: no physical parameters installed"); return -4; }
  return vjp_run(s, mode, use_pd, q, qd, tau_or_action, g_out, g_in, g_par, stream);
}

static int vjp_host(tds_b200_sim* s, int mode, int use_pd, const double* q, const double* qd,
                    const double* tau_or_action, const double* g_out, double* g_in, double* g_par) {
  if (int rc = enter_derivative_host(s)) return rc;
  const int n = s->n, ns = s->ns, n_par = g_par ? s->par.n : 0;
  int dims[2];
  tds_b200_jacobian_dims(s, mode, use_pd, dims);
  CUDA_TRY(grow_dev(&s->vjp_g, &s->vjp_g_bytes, sizeof(double) * (size_t)(dims[0] + dims[1] + n_par) * ns));
  if (int rc = put_step_inputs(s, use_pd, q, qd, tau_or_action)) return rc;
  double* gout_d = s->vjp_g;
  double* gin_d = s->vjp_g + (size_t)dims[0] * ns;
  double* gpar_d = g_par ? s->vjp_g + (size_t)(dims[0] + dims[1]) * ns : nullptr;
  CUDA_TRY(put_rows(gout_d, g_out, dims[0], n, ns, s->stream));
  CUDA_TRY(cudaMemsetAsync(gin_d, 0, sizeof(double) * (dims[1] + n_par) * ns, s->stream));
  if (int rc = vjp_run(s, mode, use_pd, s->q, s->qd, s->act, gout_d, g_in ? gin_d : nullptr, gpar_d, s->stream)) return rc;
  if (g_in) CUDA_TRY(get_rows(g_in, gin_d, dims[1], n, ns, s->stream));
  if (g_par) CUDA_TRY(get_rows(g_par, gpar_d, n_par, n, ns, s->stream));
  return 0;
}

int tds_b200_step_vjp_host(tds_b200_sim* s, int mode, int use_pd, const double* q, const double* qd,
                           const double* tau_or_action, const double* g_out, double* g_in) {
  if (int rc = vjp_check(s, mode, use_pd, q, qd, g_out, g_in)) return rc;
  return vjp_host(s, mode, use_pd, q, qd, tau_or_action, g_out, g_in, nullptr);
}

int tds_b200_step_vjp_params_host(tds_b200_sim* s, int mode, int use_pd, const double* q, const double* qd,
                                  const double* tau_or_action, const double* g_out, double* g_in, double* g_par) {
  if (int rc = vjp_check(s, mode, use_pd, q, qd, g_out, g_par)) return rc;
  if (s->par.n == 0) { set_err("parameter vjp: no physical parameters installed"); return -4; }
  return vjp_host(s, mode, use_pd, q, qd, tau_or_action, g_out, g_in, g_par);
}

// diagnostics of the VJP path: the tape capacity now in use (nodes per lane) and the environments per chunk it implies
// (a batch larger than that runs in several chunks)
int tds_b200_vjp_tape_info(const tds_b200_sim* s, int info[2]) {
  if (!s || !info) return -1;
  const size_t warps = tape_warps(s);
  info[0] = s->tape_cap;
  info[1] = (int)(warps * 32 < (size_t)1 << 30 ? warps * 32 : (size_t)1 << 30);
  return 0;
}

// ---- the step with its contact records (DESIGN.md section 7.15): the CF instances of the world-frame kernel (tds_contacts.cu).  Values
// in MODE_FULL and MODE_WORLD at the simulator's precision, on the world-frame kernel whatever kernel tds_b200_step_device would choose;
// the JVP through the Jacobian's chunk loop and the VJP by identity tangents, in MODE_FULL.
static size_t contact_rows(const tds_b200_sim* s) { return (size_t)10 * s->n_points; }

static int contacts_check(tds_b200_sim* s, int mode, int use_pd, const void* q, const void* qd, const void* tau_or_action,
                          bool derivative) {
  if (!s || !q || !qd || (use_pd && !tau_or_action)) return -1;
  if (derivative && mode != TDS_B200_MODE_FULL) { set_err("step contacts derivatives: mode FULL"); return -2; }
  if (mode != TDS_B200_MODE_FULL && mode != TDS_B200_MODE_WORLD) { set_err("step contacts: modes FULL, WORLD"); return -2; }
  if (use_pd && s->E.n_act == 0) { set_err("use_pd without tds_b200_set_env"); return -3; }
  return 0;
}

// q', qd' [dim][ns] and the records [10 n_pts][ns] fp32 of one step
static int contacts_run(tds_b200_sim* s, int mode, int use_pd, const float* q, const float* qd, const float* tau_or_action, float* q_out,
                        float* qd_out, float* contacts, cudaStream_t sm) {
  const int p = s->precision;
  if (int rc = ensure_scratch(s, p)) return rc;
  StepIO io;
  memset(&io, 0, sizeof(io));
  io.q_in = q; io.qd_in = qd; io.tau_in = tau_or_action;
  io.q_out = q_out; io.qd_out = qd_out;
  io.n = s->n; io.n_stride = s->ns;
  ParMap pmv;
  const int rc = tds_launch_contacts(&s->dm[p], &s->P, &s->E, &io, installed_par(s, &pmv), contacts, mode, use_pd, p, s->scratch, sm);
  if (rc) set_err(std::string("step contacts launch: ") + cudaGetErrorString((cudaError_t)rc));
  return rc;
}

int tds_b200_step_contacts_device(tds_b200_sim* s, int mode, int use_pd, const float* q_in, const float* qd_in, const float* tau_or_action,
                                  float* q_out, float* qd_out, float* contacts, void* stream) {
  if (int rc = contacts_check(s, mode, use_pd, q_in, qd_in, tau_or_action, false)) return rc;
  if (!q_out || !qd_out || (!contacts && s->n_points > 0)) return -1;
  return contacts_run(s, mode, use_pd, q_in, qd_in, tau_or_action, q_out, qd_out, contacts, (cudaStream_t)stream);
}

int tds_b200_step_contacts_host(tds_b200_sim* s, int mode, int use_pd, const double* q, const double* qd, const double* tau_or_action,
                                double* q_out, double* qd_out, double* contacts) {
  if (int rc = contacts_check(s, mode, use_pd, q, qd, tau_or_action, false)) return rc;
  if (!contacts && s->n_points > 0) return -1;
  if (int rc = enter_derivative_host(s)) return rc;
  const DevModel& M = s->dm[0];
  const size_t rows = contact_rows(s);
  CUDA_TRY(grow_dev(&s->jac_dev, &s->jac_dev_bytes, sizeof(float) * (rows + 1) * s->ns));
  float* rec = (float*)s->jac_dev;
  int rc = put_step_inputs(s, use_pd, q, qd, tau_or_action);
  if (!rc) rc = contacts_run(s, mode, use_pd, s->q, s->qd, s->act, s->q, s->qd, rec, s->stream);
  if (!rc) rc = get_state(s, s->q, M.n_q, q_out);
  if (!rc) rc = get_state(s, s->qd, M.n_qd, qd_out);
  if (!rc) rc = get_state(s, rec, (int)rows, contacts);
  if (rc) return rc;
  CUDA_TRY(cudaStreamSynchronize(s->stream));
  return 0;
}

static int contacts_jvp_check(tds_b200_sim* s, int mode, int use_pd, const void* q, const void* qd, const void* tau_or_action, int m,
                              const void* t_in, const void* t_par, const void* t_out) {
  if (int rc = contacts_check(s, mode, use_pd, q, qd, tau_or_action, true)) return rc;
  if (!t_out || m < 1 || (!t_in && !t_par)) return -1;
  return par_without_installed(s, t_par, "step contacts jvp: parameter tangents");
}

int tds_b200_step_contacts_jvp_device(tds_b200_sim* s, int mode, int use_pd, const float* q, const float* qd, const float* tau_or_action,
                                      int m, const double* t_in, const double* t_par, double* t_out, void* stream) {
  if (int rc = contacts_jvp_check(s, mode, use_pd, q, qd, tau_or_action, m, t_in, t_par, t_out)) return rc;
  const JvpTangents jv{t_in, t_par, m, Query::contacts};
  return jacobian_run(s, mode, use_pd, q, qd, tau_or_action, t_out, stream, false, &jv);
}

int tds_b200_step_contacts_jvp_host(tds_b200_sim* s, int mode, int use_pd, const double* q, const double* qd, const double* tau_or_action,
                                    int m, const double* t_in, const double* t_par, double* t_out) {
  if (int rc = contacts_jvp_check(s, mode, use_pd, q, qd, tau_or_action, m, t_in, t_par, t_out)) return rc;
  return step_jvp_host(s, mode, use_pd, q, qd, tau_or_action, m, t_in, t_par, t_out, Query::contacts);
}

static int contacts_vjp_check(tds_b200_sim* s, int mode, int use_pd, const void* q, const void* qd, const void* tau_or_action,
                              const void* g_out, const void* g_in, const void* g_par) {
  if (int rc = contacts_check(s, mode, use_pd, q, qd, tau_or_action, true)) return rc;
  if (!g_out || (!g_in && !g_par)) return -1;
  return par_without_installed(s, g_par, "step contacts vjp: parameter cotangents");
}

// g_in [cols][ns] (may be NULL) and g_par [k][ns] (NULL: not wanted) = <g_out, d(q' | qd' | records)> for g_out [rows][ns]
static int contacts_vjp_run(tds_b200_sim* s, int mode, int use_pd, const float* q, const float* qd, const float* tau_or_action,
                            const double* g_out, double* g_in, double* g_par, cudaStream_t sm) {
  int dims[2];
  tds_b200_jacobian_dims(s, mode, use_pd, dims);
  return vjp_by_eye(s, "step contacts", dims[1], (size_t)dims[0] + contact_rows(s), g_out, g_in, g_par, sm,
                    [&](int nd, const double* t_in, const double* t_par, double* dO) {
                      const JvpTangents jv{t_in, t_par, nd, Query::contacts};
                      return jacobian_run(s, mode, use_pd, q, qd, tau_or_action, dO, sm, false, &jv);
                    });
}

int tds_b200_step_contacts_vjp_device(tds_b200_sim* s, int mode, int use_pd, const float* q, const float* qd, const float* tau_or_action,
                                      const double* g_out, double* g_in, double* g_par, void* stream) {
  if (int rc = contacts_vjp_check(s, mode, use_pd, q, qd, tau_or_action, g_out, g_in, g_par)) return rc;
  return contacts_vjp_run(s, mode, use_pd, q, qd, tau_or_action, g_out, g_in, g_par, (cudaStream_t)stream);
}

int tds_b200_step_contacts_vjp_host(tds_b200_sim* s, int mode, int use_pd, const double* q, const double* qd, const double* tau_or_action,
                                    const double* g_out, double* g_in, double* g_par) {
  if (int rc = contacts_vjp_check(s, mode, use_pd, q, qd, tau_or_action, g_out, g_in, g_par)) return rc;
  if (int rc = enter_derivative_host(s)) return rc;
  const int n = s->n, ns = s->ns, k = g_par ? s->par.n : 0;
  int dims[2];
  tds_b200_jacobian_dims(s, mode, use_pd, dims);
  const size_t rows = (size_t)dims[0] + contact_rows(s);
  // g_out | g_in | g_par
  CUDA_TRY(grow_dev(&s->vjp_g, &s->vjp_g_bytes, sizeof(double) * (rows + dims[1] + k + 1) * ns));
  double* g_d = s->vjp_g + rows * ns;
  if (int rc = put_step_inputs(s, use_pd, q, qd, tau_or_action)) return rc;
  CUDA_TRY(put_rows(s->vjp_g, g_out, rows, n, ns, s->stream));
  if (int rc = contacts_vjp_run(s, mode, use_pd, s->q, s->qd, s->act, s->vjp_g, g_d, g_par ? g_d + (size_t)dims[1] * ns : nullptr,
                                s->stream))
    return rc;
  CUDA_TRY(get_parts<double>({{g_in, (size_t)dims[1]}, {g_par, (size_t)k}}, g_d, n, ns, s->stream));
  return 0;
}

// ---- the step with external wrenches (DESIGN.md section 7.18): the EXT instances of the world-frame kernel (tds_wrench.cu).  Values in
// MODE_FD, MODE_NOCONTACT and MODE_FULL at the simulator's precision, on the world-frame kernel whatever kernel tds_b200_step_device would
// choose; the JVP through the Jacobian's chunk loop and the VJP by identity tangents.  The point table is checked as for the kinematics
// (kin_check); the wrench columns follow the step's columns (tds_b200_jacobian_dims) and precede the installed parameters.
static int wrench_check(tds_b200_sim* s, int mode, int use_pd, const void* q, const void* qd, const void* tau_or_action, int K,
                        const int* links, const double* local, const void* W) {
  if (int rc = kin_check(s, q, K, links, local)) return rc;
  if (!qd || (use_pd && !tau_or_action) || (K > 0 && !W)) return -1;
  if (mode == TDS_B200_MODE_WORLD) { set_err("step wrench: modes FD, NOCONTACT, FULL"); return -2; }
  if (use_pd && s->E.n_act == 0) { set_err("use_pd without tds_b200_set_env"); return -3; }
  return 0;
}

// q', qd' [dim][ns] (MODE_NOCONTACT, MODE_FULL) or qdd [n_qd][ns] (MODE_FD) fp32 of one step with the wrenches W [6K][ns] fp32
static int wrench_run(tds_b200_sim* s, int mode, int use_pd, const float* q, const float* qd, const float* tau_or_action, const TdsExtCall* xc,
                      float* q_out, float* qd_out, float* qdd_out, cudaStream_t sm) {
  const int p = s->precision;
  CUDA_TRY(grow_dev(&s->jac_scratch, &s->jac_scratch_bytes, wrench_arena_bytes(s, s->dm[p], p == TDS_B200_PREC_F64 ? 8 : 4)));
  StepIO io;
  memset(&io, 0, sizeof(io));
  io.q_in = q; io.qd_in = qd; io.tau_in = tau_or_action;
  io.q_out = q_out; io.qd_out = qd_out; io.qdd_out = qdd_out;
  io.n = s->n; io.n_stride = s->ns;
  ParMap pmv;
  const int rc = tds_launch_wrench(&s->dm[p], &s->P, &s->E, &io, installed_par(s, &pmv), xc, mode, use_pd, p, s->jac_scratch, sm);
  if (rc) set_err(std::string("step wrench launch: ") + cudaGetErrorString((cudaError_t)rc));
  return rc;
}

// the outputs a mode needs: qdd in MODE_FD, q' and qd' otherwise
static int wrench_out_check(int mode, const void* q_out, const void* qd_out, const void* qdd_out) {
  if (mode == TDS_B200_MODE_FD ? !qdd_out : (!q_out || !qd_out)) return -1;
  return 0;
}

int tds_b200_step_wrench_device(tds_b200_sim* s, int mode, int use_pd, const float* q_in, const float* qd_in, const float* tau_or_action,
                                int K, const int* links, const double* local, const float* W, float* q_out, float* qd_out, float* qdd_out,
                                void* stream) {
  if (int rc = wrench_check(s, mode, use_pd, q_in, qd_in, tau_or_action, K, links, local, W)) return rc;
  if (int rc = wrench_out_check(mode, q_out, qd_out, qdd_out)) return rc;
  const TdsExtCall xc{K, links, local, W, nullptr};
  return wrench_run(s, mode, use_pd, q_in, qd_in, tau_or_action, &xc, q_out, qd_out, qdd_out, (cudaStream_t)stream);
}

// W [n][K][6] fp64 -> s->wrench_dev [6K][ns] fp32, with the step's inputs
static int put_wrench_inputs(tds_b200_sim* s, int use_pd, const double* q, const double* qd, const double* tau_or_action, int K,
                             const double* W) {
  if (int rc = put_step_inputs(s, use_pd, q, qd, tau_or_action)) return rc;
  CUDA_TRY(grow_dev(&s->wrench_dev, &s->wrench_dev_bytes, sizeof(float) * (size_t)(6 * K + 1) * s->ns));
  if (K == 0) return 0;
  if (int rc = ensure_stage(s, sizeof(double) * s->n * 6 * K)) return rc;
  return put_state(s, W, 6 * K, s->wrench_dev);
}

int tds_b200_step_wrench_host(tds_b200_sim* s, int mode, int use_pd, const double* q, const double* qd, const double* tau_or_action, int K,
                              const int* links, const double* local, const double* W, double* q_out, double* qd_out, double* qdd_out) {
  if (int rc = wrench_check(s, mode, use_pd, q, qd, tau_or_action, K, links, local, W)) return rc;
  if (int rc = wrench_out_check(mode, q_out, qd_out, qdd_out)) return rc;
  if (int rc = enter_derivative_host(s)) return rc;
  const DevModel& M = s->dm[0];
  int rc = put_wrench_inputs(s, use_pd, q, qd, tau_or_action, K, W);
  const TdsExtCall xc{K, links, local, s->wrench_dev, nullptr};
  if (!rc) rc = wrench_run(s, mode, use_pd, s->q, s->qd, s->act, &xc, s->q, s->qd, s->qdd, s->stream);
  if (!rc && mode == TDS_B200_MODE_FD) rc = get_state(s, s->qdd, M.n_qd, qdd_out);
  if (!rc && mode != TDS_B200_MODE_FD) rc = get_state(s, s->q, M.n_q, q_out);
  if (!rc && mode != TDS_B200_MODE_FD) rc = get_state(s, s->qd, M.n_qd, qd_out);
  if (rc) return rc;
  CUDA_TRY(cudaStreamSynchronize(s->stream));
  return 0;
}

static int wrench_jvp_check(tds_b200_sim* s, int mode, int use_pd, const void* q, const void* qd, const void* tau_or_action, int K,
                            const int* links, const double* local, const void* W, int m, const void* t_in, const void* t_W, const void* t_par,
                            const void* t_out) {
  if (int rc = wrench_check(s, mode, use_pd, q, qd, tau_or_action, K, links, local, W)) return rc;
  if (!t_out || m < 1 || (!t_in && !t_W && !t_par)) return -1;
  return par_without_installed(s, t_par, "step wrench jvp: parameter tangents");
}

int tds_b200_step_wrench_jvp_device(tds_b200_sim* s, int mode, int use_pd, const float* q, const float* qd, const float* tau_or_action, int K,
                                    const int* links, const double* local, const float* W, int m, const double* t_in, const double* t_W,
                                    const double* t_par, double* t_out, void* stream) {
  if (int rc = wrench_jvp_check(s, mode, use_pd, q, qd, tau_or_action, K, links, local, W, m, t_in, t_W, t_par, t_out)) return rc;
  const TdsExtCall xc{K, links, local, W, t_W};
  JvpTangents jv{t_in, t_par, m, Query::wrench};
  jv.ext = &xc;
  return jacobian_run(s, mode, use_pd, q, qd, tau_or_action, t_out, stream, false, &jv);
}

int tds_b200_step_wrench_jvp_host(tds_b200_sim* s, int mode, int use_pd, const double* q, const double* qd, const double* tau_or_action,
                                  int K, const int* links, const double* local, const double* W, int m, const double* t_in, const double* t_W,
                                  const double* t_par, double* t_out) {
  if (int rc = wrench_jvp_check(s, mode, use_pd, q, qd, tau_or_action, K, links, local, W, m, t_in, t_W, t_par, t_out)) return rc;
  if (int rc = enter_derivative_host(s)) return rc;
  const int n = s->n, ns = s->ns, k = s->par.n;
  int dims[2];
  tds_b200_jacobian_dims(s, mode, use_pd, dims);
  // tangents: host [n][dim][m] <-> device [dim * m][ns]; t_in | t_W | t_par | t_out
  const size_t ti = (size_t)(t_in ? dims[1] : 0) * m, tw = (size_t)(t_W ? 6 * K : 0) * m, tp = (size_t)(t_par ? k : 0) * m,
               to = (size_t)dims[0] * m;
  CUDA_TRY(grow_dev(&s->jac_dev, &s->jac_dev_bytes, sizeof(double) * (ti + tw + tp + to) * ns));
  if (int rc = put_wrench_inputs(s, use_pd, q, qd, tau_or_action, K, W)) return rc;
  double* tout_d = s->jac_dev + (ti + tw + tp) * ns;
  CUDA_TRY(put_parts<double>(s->jac_dev, {{t_in, ti}, {t_W, tw}, {t_par, tp}, {nullptr, to}}, n, ns, s->stream));
  const TdsExtCall xc{K, links, local, s->wrench_dev, t_W ? s->jac_dev + ti * ns : nullptr};
  JvpTangents jv{t_in ? s->jac_dev : nullptr, t_par ? s->jac_dev + (ti + tw) * ns : nullptr, m, Query::wrench};
  jv.ext = &xc;
  if (int rc = jacobian_run(s, mode, use_pd, s->q, s->qd, s->act, tout_d, s->stream, false, &jv)) return rc;
  CUDA_TRY(get_rows(t_out, tout_d, to, n, ns, s->stream));
  return 0;
}

static int wrench_vjp_check(tds_b200_sim* s, int mode, int use_pd, const void* q, const void* qd, const void* tau_or_action, int K,
                            const int* links, const double* local, const void* W, const void* g_out, const void* g_in, const void* g_W,
                            const void* g_par) {
  if (int rc = wrench_check(s, mode, use_pd, q, qd, tau_or_action, K, links, local, W)) return rc;
  if (!g_out || (!g_in && !g_W && !g_par)) return -1;
  return par_without_installed(s, g_par, "step wrench vjp: parameter cotangents");
}

// g_inw [cols + 6K][ns] (the step's inputs, then the wrenches) and g_par [k][ns] (NULL: not wanted) = <g_out, d(q' | qd', or qdd)> for
// g_out [rows][ns]; the wrench tangents are the identity tangents' rows behind the step's columns
static int wrench_vjp_run(tds_b200_sim* s, int mode, int use_pd, const float* q, const float* qd, const float* tau_or_action, int K,
                          const int* links, const double* local, const float* W, const double* g_out, double* g_inw, double* g_par,
                          cudaStream_t sm) {
  int dims[2];
  tds_b200_jacobian_dims(s, mode, use_pd, dims);
  const size_t ns = s->ns;
  return vjp_by_eye(s, "step wrench", dims[1] + 6 * K, dims[0], g_out, g_inw, g_par, sm,
                    [&](int nd, const double* t_in, const double* t_par, double* dO) {
                      const TdsExtCall xc{K, links, local, W, t_in + (size_t)dims[1] * nd * ns};
                      JvpTangents jv{t_in, t_par, nd, Query::wrench};
                      jv.ext = &xc;
                      return jacobian_run(s, mode, use_pd, q, qd, tau_or_action, dO, sm, false, &jv);
                    });
}

int tds_b200_step_wrench_vjp_device(tds_b200_sim* s, int mode, int use_pd, const float* q, const float* qd, const float* tau_or_action, int K,
                                    const int* links, const double* local, const float* W, const double* g_out, double* g_in, double* g_W,
                                    double* g_par, void* stream) {
  if (int rc = wrench_vjp_check(s, mode, use_pd, q, qd, tau_or_action, K, links, local, W, g_out, g_in, g_W, g_par)) return rc;
  int dims[2];
  tds_b200_jacobian_dims(s, mode, use_pd, dims);
  cudaStream_t sm = (cudaStream_t)stream;
  // g_in | g_W as one array for the contraction
  CUDA_TRY(grow_dev(&s->vjp_g, &s->vjp_g_bytes, sizeof(double) * (size_t)(dims[1] + 6 * K) * s->ns));
  if (int rc = wrench_vjp_run(s, mode, use_pd, q, qd, tau_or_action, K, links, local, W, g_out, s->vjp_g, g_par, sm)) return rc;
  CUDA_TRY(get_parts_d2d<double>({{g_in, (size_t)dims[1]}, {g_W, (size_t)6 * K}}, s->vjp_g, s->ns, sm));
  return 0;
}

int tds_b200_step_wrench_vjp_host(tds_b200_sim* s, int mode, int use_pd, const double* q, const double* qd, const double* tau_or_action,
                                  int K, const int* links, const double* local, const double* W, const double* g_out, double* g_in,
                                  double* g_W, double* g_par) {
  if (int rc = wrench_vjp_check(s, mode, use_pd, q, qd, tau_or_action, K, links, local, W, g_out, g_in, g_W, g_par)) return rc;
  if (int rc = enter_derivative_host(s)) return rc;
  const int n = s->n, ns = s->ns, k = g_par ? s->par.n : 0;
  int dims[2];
  tds_b200_jacobian_dims(s, mode, use_pd, dims);
  // g_out | g_in | g_W | g_par
  CUDA_TRY(grow_dev(&s->vjp_g, &s->vjp_g_bytes, sizeof(double) * ((size_t)dims[0] + dims[1] + 6 * K + k + 1) * ns));
  double* g_d = s->vjp_g + (size_t)dims[0] * ns;
  if (int rc = put_wrench_inputs(s, use_pd, q, qd, tau_or_action, K, W)) return rc;
  CUDA_TRY(put_rows(s->vjp_g, g_out, dims[0], n, ns, s->stream));
  if (int rc = wrench_vjp_run(s, mode, use_pd, s->q, s->qd, s->act, K, links, local, s->wrench_dev, s->vjp_g, g_d,
                              g_par ? g_d + (size_t)(dims[1] + 6 * K) * ns : nullptr, s->stream))
    return rc;
  CUDA_TRY(get_parts<double>({{g_in, (size_t)dims[1]}, {g_W, (size_t)6 * K}, {g_par, (size_t)k}}, g_d, n, ns, s->stream));
  return 0;
}

int tds_b200_step_host(tds_b200_sim* s, int mode, int use_pd, const double* q, const double* qd,
                       const double* tau_or_action, double* q_out, double* qd_out, double* qdd_out,
                       double* contact_dist) {
  if (!s || !q || !qd) return -1;
  CUDA_TRY(cudaSetDevice(s->device));
  const DevModel& M = s->dm[0];
  int rc = put_step_inputs(s, use_pd, q, qd, tau_or_action);
  if (!rc) rc = tds_b200_step_device(s, mode, use_pd, s->q, s->qd, s->act, s->q, s->qd, s->qdd, nullptr, nullptr,
                                     contact_dist ? s->cdist : nullptr, nullptr, s->stream);
  if (!rc) rc = get_state(s, s->q, M.n_q, q_out);
  if (!rc) rc = get_state(s, s->qd, M.n_qd, qd_out);
  if (!rc && mode == TDS_B200_MODE_FD) rc = get_state(s, s->qdd, M.n_qd, qdd_out);
  if (!rc) rc = get_state(s, s->cdist, s->n_points, contact_dist);
  if (rc) return rc;
  CUDA_TRY(cudaStreamSynchronize(s->stream));
  CUDA_TRY(cudaGetLastError());
  return 0;
}

static IntegrateTable integrate_table(const tds_b200_sim* s) {
  const DevModel& M = s->dm[0];
  IntegrateTable T;
  memset(&T, 0, sizeof(T));
  T.n_links = M.n_links; T.floating = M.floating; T.n_q = M.n_q; T.n_qd = M.n_qd;
  for (int i = 0; i < M.n_links; ++i) {
    T.fixed[i] = (M.flags[i] & TDS_LF_FIXED) ? 1 : 0;
    T.q_idx[i] = (signed char)(T.fixed[i] ? 0 : M.q_idx[i]); T.qd_idx[i] = (signed char)(T.fixed[i] ? 0 : M.qd_idx[i]);
  }
  return T;
}

int tds_b200_integrate_euler_device(tds_b200_sim* s, float* q, float* qd, const float* qdd, void* stream) {
  if (!s || !q || !qd) return -1;
  if (s->dm[0].n_sph) { set_err("stand-alone integrate_euler: spherical joints are integrated by the step kernel only"); return -3; }
  const int T = 128, B = (s->n + T - 1) / T;
  integrate_euler_kernel<<<B, T, 0, (cudaStream_t)stream>>>(q, qd, qdd, s->P.dt, integrate_table(s), 1, s->n, s->ns);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int tds_b200_integrate_euler_qdd_device(tds_b200_sim* s, float* qd, const float* qdd, void* stream) {
  if (!s || !qd || !qdd) return -1;
  const int T = 128, B = (s->n + T - 1) / T;
  integrate_euler_kernel<<<B, T, 0, (cudaStream_t)stream>>>(qd, qd, qdd, s->P.dt, integrate_table(s), 0, s->n, s->ns);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

static int write_tuples(const ContactCandTable& T, int* tuples, int cap) {
  for (int c = 0; c < T.n_points && c < cap && tuples; ++c) {
    tuples[4 * c + 0] = T.body_a[c]; tuples[4 * c + 1] = T.link_a[c];
    tuples[4 * c + 2] = T.body_b[c]; tuples[4 * c + 3] = T.link_b[c];
  }
  return T.n_points;
}

static int write_tuples6(const ContactCandTable& T, int* tuples, int cap) {
  for (int c = 0; c < T.n_points && c < cap && tuples; ++c) {
    tuples[6 * c + 0] = T.body_a[c]; tuples[6 * c + 1] = T.link_a[c]; tuples[6 * c + 2] = T.geom_a[c];
    tuples[6 * c + 3] = T.body_b[c]; tuples[6 * c + 4] = T.link_b[c]; tuples[6 * c + 5] = T.geom_b[c];
  }
  return T.n_points;
}

// (mb_a, link_a, geom_a, mb_b, link_b, geom_b) per candidate: the loop indices i, ii, iii, j, jj, jjj of
// World::compute_contacts_multi_body_internal (src/world.hpp:212-240) at which the point is emitted.
int tds_b200_model_contact_tuples(const double* model, int n_model, int* tuples, int cap) {
  if (!model) { set_err("null model"); return -1; }
  DevModel* D = new DevModel;
  const int rc = tds_build_dev_model(model, n_model, D);
  ContactCandTable T;
  if (rc == 0) T = make_cand_table(*D);
  delete D;
  if (rc) { set_err(std::string("unsupported model: ") + tds_model_error(rc)); return rc; }
  return write_tuples6(T, tuples, cap);
}

int tds_b200_contact_tuples(const tds_b200_sim* s, int* tuples, int cap) {
  if (!s) return -1;
  return write_tuples6(s->cand, tuples, cap);
}

// Host-only variant (no GPU needed): the candidate list of a flat model.
int tds_b200_model_contact_pairs(const double* model, int n_model, int* tuples, int cap) {
  if (!model) { set_err("null model"); return -1; }
  DevModel* D = new DevModel;
  const int rc = tds_build_dev_model(model, n_model, D);
  ContactCandTable T;
  if (rc == 0) T = make_cand_table(*D);
  delete D;
  if (rc) { set_err(std::string("unsupported model: ") + tds_model_error(rc)); return rc; }
  return write_tuples(T, tuples, cap);
}

int tds_b200_contact_pairs(const tds_b200_sim* s, int* tuples, int cap) {
  if (!s) return -1;
  return write_tuples(s->cand, tuples, cap);
}

int tds_b200_contact_list_device(tds_b200_sim* s, const float* contact_dist, int* count, int* links, void* stream) {
  if (!s || !contact_dist || !count || !links) return -1;
  if (s->cand.n_points == 0) return 0;
  const int T = 128, B = (s->n + T - 1) / T;
  contact_list_kernel<<<B, T, 0, (cudaStream_t)stream>>>(contact_dist, s->cand, s->P.keep_all_points, count, links, nullptr, s->n, s->ns);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int tds_b200_contact_list_host(tds_b200_sim* s, int* count, int* links) {
  if (!s || !count) return -1;
  CUDA_TRY(cudaSetDevice(s->device));
  const int n = s->n, ns = s->ns, np = s->cand.n_points;
  if (np == 0) { for (int e = 0; e < n; ++e) count[e] = 0; return 0; }
  CUDA_TRY(grow_dev(&s->c_count, &s->c_count_bytes, sizeof(int) * ns));
  CUDA_TRY(grow_dev(&s->c_links, &s->c_links_bytes, sizeof(int) * (size_t)ns * 2 * np));
  if (int rc = tds_b200_contact_list_device(s, s->cdist, s->c_count, s->c_links, s->stream)) return rc;
  CUDA_TRY(get_rows(count, s->c_count, 1, n, ns, s->stream));
  if (links) CUDA_TRY(get_rows(links, s->c_links, 2 * np, n, ns, s->stream));
  return 0;
}

int tds_b200_contact_list_candidates_host(tds_b200_sim* s, int* count, int* cand) {
  if (!s || !count || !cand) return -1;
  CUDA_TRY(cudaSetDevice(s->device));
  const int n = s->n, ns = s->ns, np = s->cand.n_points;
  if (np == 0) { for (int e = 0; e < n; ++e) count[e] = 0; return 0; }
  CUDA_TRY(grow_dev(&s->c_count, &s->c_count_bytes, sizeof(int) * ns));
  CUDA_TRY(grow_dev(&s->c_links, &s->c_links_bytes, sizeof(int) * (size_t)ns * 2 * np));
  CUDA_TRY(grow_dev(&s->c_cand, &s->c_cand_bytes, sizeof(int) * (size_t)ns * np));
  const int T = 128, B = (n + T - 1) / T;
  contact_list_kernel<<<B, T, 0, s->stream>>>(s->cdist, s->cand, s->P.keep_all_points, s->c_count, s->c_links, s->c_cand, n, ns);
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(get_rows(count, s->c_count, 1, n, ns, s->stream));
  CUDA_TRY(get_rows(cand, s->c_cand, np, n, ns, s->stream));
  return 0;
}

int tds_b200_env_set_state_host(tds_b200_sim* s, const double* q, const double* qd) {
  if (!s) return -1;
  CUDA_TRY(cudaSetDevice(s->device));
  int rc = put_q(s, q);
  if (!rc) rc = put_state(s, qd, s->dm[0].n_qd, s->qd);
  if (rc) return rc;
  CUDA_TRY(cudaStreamSynchronize(s->stream));
  return 0;
}

int tds_b200_env_get_state_host(tds_b200_sim* s, double* q, double* qd) {
  if (!s) return -1;
  CUDA_TRY(cudaSetDevice(s->device));
  const int rc = get_state(s, s->q, s->dm[0].n_q, q);
  return rc ? rc : get_state(s, s->qd, s->dm[0].n_qd, qd);
}

int tds_b200_env_step_device(tds_b200_sim* s, const float* actions, float* reward, float* done, void* stream) {
  if (!s) return -1;
  return tds_b200_step_device(s, TDS_B200_MODE_FULL, 1, s->q, s->qd, actions, s->q, s->qd, nullptr, reward, done,
                              nullptr, nullptr, stream);
}

int tds_b200_num_visuals(const tds_b200_sim* s) { return s ? s->vis.n_vis : -1; }

int tds_b200_env_step_visual_device(tds_b200_sim* s, const float* actions, float* reward, float* done, float* positions,
                                    float* orientations, void* stream) {
  if (!s || !positions || !orientations) return -1;
  if (s->vis.n_vis <= 0) { set_err("model has no link visuals"); return -2; }
  int rc = tds_b200_step_device(s, TDS_B200_MODE_FULL, 1, s->q, s->qd, actions, s->q, s->qd, nullptr, reward, done, nullptr,
                                s->link_xf, stream);
  if (rc) return rc;
  const int T = 128, B = (s->n + T - 1) / T;
  pack_visual_instances_kernel<<<dim3(B, s->vis.n_vis), T, 0, (cudaStream_t)stream>>>(s->vis, s->link_xf, (float4*)positions,
                                                                                     (float4*)orientations, s->n, s->ns);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

static int ensure_env_layer(tds_b200_sim* s) {
  if (s->rq) return 0;
  const DevModel& M = s->dm[0];
  const size_t ns = s->ns;
  CUDA_TRY(cudaMalloc((void**)&s->rq, sizeof(float) * ns * (M.n_q > 0 ? M.n_q : 1)));
  CUDA_TRY(cudaMalloc((void**)&s->rqd, sizeof(float) * ns * (M.n_qd > 0 ? M.n_qd : 1)));
  CUDA_TRY(cudaMalloc((void**)&s->zero_act, sizeof(float) * ns * TDS_MAX_ACT));
  CUDA_TRY(cudaMemset(s->zero_act, 0, sizeof(float) * ns * TDS_MAX_ACT));
  CUDA_TRY(cudaMalloc((void**)&s->pol_act, sizeof(float) * ns * TDS_MAX_ACT));
  CUDA_TRY(cudaMalloc((void**)&s->sticky, sizeof(float) * ns));
  CUDA_TRY(cudaMalloc((void**)&s->r_total, sizeof(float) * ns));
  CUDA_TRY(cudaMalloc((void**)&s->r_steps, sizeof(int) * ns));
  CUDA_TRY(cudaMalloc((void**)&s->act_qidx, sizeof(int) * TDS_MAX_ACT));
  return 0;
}

int tds_b200_env_reset_device(tds_b200_sim* s, const float* mask, const float* noise, float noise_amp, unsigned long long seed,
                              int settle_steps, void* stream) {
  if (!s) return -1;
  if (s->E.n_act == 0) { set_err("env reset without tds_b200_set_env"); return -3; }
  CUDA_TRY(cudaSetDevice(s->device));
  int rc = ensure_env_layer(s);
  if (rc) return rc;
  const DevModel& M = s->dm[0];
  cudaStream_t sm = stream ? (cudaStream_t)stream : s->stream;   // NULL: the simulator's own stream (as the host paths)
  if (!s->act_qidx_valid) {   // once per actuator map (synchronous: keeps the reset itself capturable into a CUDA graph)
    int qidx[TDS_MAX_ACT];
    for (int a = 0; a < s->E.n_act; ++a) qidx[a] = M.q_idx[s->E.act_link[a]];
    CUDA_TRY(cudaMemcpy(s->act_qidx, qidx, sizeof(int) * s->E.n_act, cudaMemcpyHostToDevice));
    s->act_qidx_valid = true;
  }
  const int T = 128, B = (s->n + T - 1) / T;
  env_reset_fill_kernel<<<B, T, 0, sm>>>(s->rq, s->rqd, noise, noise_amp, seed, s->E, M.n_q, M.n_qd, s->act_qidx, s->n, s->ns);
  // settle with zero actions on the staging copy (laikago_environment2.h:92-110); no auto-reset inside
  const int saved_auto = s->E.auto_reset;
  s->E.auto_reset = 0;
  for (int i = 0; i < settle_steps && rc == 0; ++i)
    rc = tds_b200_step_device(s, TDS_B200_MODE_FULL, 1, s->rq, s->rqd, s->zero_act, s->rq, s->rqd, nullptr, nullptr, nullptr,
                              nullptr, nullptr, sm);
  s->E.auto_reset = saved_auto;
  if (rc) return rc;
  env_select_kernel<<<B, T, 0, sm>>>(mask, s->rq, s->rqd, s->q, s->qd, M.n_q, M.n_qd, s->n, s->ns);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int tds_b200_ars_perturb_device(tds_b200_sim* s, const float* w, const float* deltas, float scale, float* params, int n_params,
                                void* stream) {
  if (!s || !w || !deltas || !params || n_params <= 0) return -1;
  const int T = 128, B = (s->n + T - 1) / T;
  ars_perturb_kernel<<<dim3(B, n_params), T, 0, (cudaStream_t)stream>>>(w, deltas, scale, params, s->n, s->ns);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int tds_b200_ars_update_device(tds_b200_sim* s, float* w, const float* deltas, const float* r_pos, const float* r_neg,
                               float delta_std, float step_size, int n_params, void* stream) {
  if (!s || !w || !deltas || !r_pos || !r_neg || n_params <= 0) return -1;
  ars_update_kernel<<<n_params, 256, 0, (cudaStream_t)stream>>>(w, deltas, r_pos, r_neg, delta_std, step_size, s->n, s->ns);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int tds_b200_env_set_obs_stats(tds_b200_sim* s, float* stats) {
  if (!s) return -1;
  s->obs_stats = stats;
  return 0;
}

int tds_b200_env_rollout_device(tds_b200_sim* s, const float* policy, int n_params, int rollout_length, float shift,
                                float* total_rewards, int* steps, void* stream) {
  if (!s || !policy || !total_rewards || !steps) return -1;
  if (s->E.n_act == 0) { set_err("rollout without tds_b200_set_env"); return -3; }
  const DevModel& M = s->dm[0];
  if (n_params != s->E.n_act * (M.n_q + M.n_qd) + s->E.n_act) { set_err("policy size must be n_act * (n_q + n_qd) + n_act"); return -2; }
  CUDA_TRY(cudaSetDevice(s->device));
  int rc = ensure_env_layer(s);
  if (rc) return rc;
  cudaStream_t sm = stream ? (cudaStream_t)stream : s->stream;
  const int T = 128, B = (s->n + T - 1) / T;
  rollout_init_kernel<<<B, T, 0, sm>>>(s->sticky, total_rewards, steps, s->n);
  const int saved_auto = s->E.auto_reset;
  s->E.auto_reset = 0;   // an episode ends at done (ars_vectorized_worker.h:121-133)
  for (int r = 0; r < rollout_length && rc == 0; ++r) {
    policy_linear_kernel<<<dim3(B, s->E.n_act), T, 0, sm>>>(s->q, s->qd, policy, s->pol_act, M.n_q, M.n_qd, s->E.n_act, s->n, s->ns);
    if (s->obs_stats) obs_stat_push_kernel<<<dim3(B, M.n_q + M.n_qd), T, 0, sm>>>(s->q, s->qd, s->obs_stats, M.n_q, M.n_qd, s->n, s->ns);
    rc = tds_b200_step_device(s, TDS_B200_MODE_FULL, 1, s->q, s->qd, s->pol_act, s->q, s->qd, nullptr, s->reward, s->done, nullptr,
                              nullptr, sm);
    rollout_accum_kernel<<<B, T, 0, sm>>>(s->reward, s->done, shift, s->sticky, total_rewards, steps, s->n);
  }
  s->E.auto_reset = saved_auto;
  if (rc) return rc;
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int tds_b200_env_rollout_host(tds_b200_sim* s, const double* policy, int n_params, int rollout_length, double shift,
                              const double* noise, double noise_amp, unsigned long long seed, int settle_steps,
                              double* total_rewards, int* steps) {
  if (!s || !policy) return -1;
  CUDA_TRY(cudaSetDevice(s->device));
  int rc = ensure_env_layer(s);
  if (rc) return rc;
  const int n = s->n, ns = s->ns, na = s->E.n_act;
  cudaStream_t sm = s->stream;
  const size_t rows = (size_t)n_params > (size_t)na ? (size_t)n_params : (size_t)na;
  CUDA_TRY(grow_dev(&s->pol_params, &s->pol_params_bytes, sizeof(float) * rows * ns));
  rc = ensure_stage(s, sizeof(double) * (size_t)n * rows);
  if (!rc && noise) rc = put_state(s, noise, na, s->pol_params);   // [n][n_act] -> [n_act][ns]
  if (!rc) rc = tds_b200_env_reset_device(s, nullptr, noise ? s->pol_params : nullptr, (float)noise_amp, seed, settle_steps, sm);
  if (!rc) rc = put_state(s, policy, n_params, s->pol_params);
  if (!rc) rc = tds_b200_env_rollout_device(s, s->pol_params, n_params, rollout_length, (float)shift, s->r_total, s->r_steps, sm);
  if (rc) return rc;
  std::vector<float> tot(n);
  CUDA_TRY(cudaMemcpyAsync(tot.data(), s->r_total, sizeof(float) * n, cudaMemcpyDeviceToHost, sm));
  if (steps) CUDA_TRY(cudaMemcpyAsync(steps, s->r_steps, sizeof(int) * n, cudaMemcpyDeviceToHost, sm));
  CUDA_TRY(cudaStreamSynchronize(sm));
  if (total_rewards) for (int i = 0; i < n; ++i) total_rewards[i] = (double)tot[i];
  return 0;
}

// Profiling aid (not part of the drop-in surface): enable per-warp clock64() stamps at the phase
// boundaries of the step kernel; out (host) receives [n_warps][16] stamps of the last step.
int tds_b200_get_precision(const tds_b200_sim* s) { return s ? s->precision : -1; }

const char* tds_b200_kernel_name(const tds_b200_sim* s) {
  static const char* names[5] = {"", "tds_stepw_kernel (common frame, lane per environment)",
                                 "tds_stept_kernel (lane team per environment)", "tds_stepr_kernel (warp per tree role)",
                                 "tds_step_spec_kernel (warp per tree role, model-specialised)"};
  return (s && s->kernel >= 0 && s->kernel <= 4) ? names[s->kernel] : "";
}

int tds_b200_debug_phase_clocks(tds_b200_sim* s, int enable, long long* out_host, int cap_warps) {
  if (!s) return -1;
  const int nw = s->ns / (32 / TDS_TEAM_T);   // team kernel: 8 environments per warp
  if (enable && !s->phase_clk) {
    CUDA_TRY(cudaMalloc((void**)&s->phase_clk, sizeof(long long) * 16 * nw));
    CUDA_TRY(cudaMemset(s->phase_clk, 0, sizeof(long long) * 16 * nw));
  }
  if (out_host && s->phase_clk) {
    CUDA_TRY(cudaDeviceSynchronize());
    CUDA_TRY(cudaMemcpy(out_host, s->phase_clk, sizeof(long long) * 16 * (nw < cap_warps ? nw : cap_warps), cudaMemcpyDeviceToHost));
  }
  if (!enable && s->phase_clk) { cudaFree(s->phase_clk); s->phase_clk = nullptr; }
  return nw;
}

// Profiling aid: the launches enqueued from now on write their stamps to the caller's device buffer ([n_warps][16], see
// tds_b200_debug_phase_clocks for n_warps) instead; null returns to the library's own record.  One buffer per launch
// keeps the stamps of every step of a captured sequence (scripts/step_gaps.py).
int tds_b200_debug_phase_clocks_device(tds_b200_sim* s, long long* dev) {
  if (!s) return -1;
  s->phase_clk_dev = dev;
  return 0;
}

void* tds_b200_stream(tds_b200_sim* s) { return s ? (void*)s->stream : nullptr; }
float* tds_b200_env_q(tds_b200_sim* s) { return s ? s->q : nullptr; }
float* tds_b200_env_qd(tds_b200_sim* s) { return s ? s->qd : nullptr; }

int tds_b200_env_step_host(tds_b200_sim* s, const float* actions, float* obs, float* rewards, float* dones) {
  if (!s || !actions) return -1;
  CUDA_TRY(cudaSetDevice(s->device));
  const DevModel& M = s->dm[0];
  const int n = s->n, ns = s->ns, na = s->E.n_act, nobs = M.n_q + M.n_qd;
  // device staging: actions AoS in | obs AoS out | reward | done
  const size_t in_b = sizeof(float) * (size_t)n * na, obs_b = sizeof(float) * (size_t)n * nobs;
  // obs | rewards | dones adjacent in the caller's memory: pack them on the device and copy once
  const bool packed = obs && rewards == obs + (size_t)n * nobs && dones == rewards + n;
  int rc = ensure_stage(s, in_b + obs_b + sizeof(float) * 2 * (size_t)n);
  if (rc) return rc;
  float* d_in = (float*)s->stage_dev;
  float* d_obs = (float*)((char*)s->stage_dev + in_b);
  cudaStream_t sm = s->stream;
  const int T = 128, B = (n + T - 1) / T;
  // the specialised kernel reads environment-major actions and writes the observation block itself
  const bool direct = s->kernel_req == 4 && s->spec_ok && s->P.contact_model == 0 && s->par.n == 0 && tds_spec_smem_bytes(s->spec_idx, s->precision) <= (size_t)s->max_smem_optin;
  auto enqueue = [&]() -> int {
    CUDA_TRY(cudaMemcpyAsync(d_in, actions, in_b, cudaMemcpyHostToDevice, sm));
    if (direct) {
      s->io_act_aos = d_in; s->io_obs_aos = obs ? d_obs : nullptr; s->io_obs_tail = (obs && packed) ? d_obs + (size_t)n * nobs : nullptr;
    } else aos_to_soa_kernel<float><<<B, T, 0, sm>>>(d_in, na, 0, s->act, na, n, ns);
    int r = tds_b200_step_device(s, TDS_B200_MODE_FULL, 1, s->q, s->qd, s->act, s->q, s->qd, nullptr, s->reward, s->done,
                                 nullptr, nullptr, sm);
    s->io_act_aos = nullptr; s->io_obs_aos = nullptr; s->io_obs_tail = nullptr;
    if (r) return r;
    if (obs && direct) {
      CUDA_TRY(cudaMemcpyAsync(obs, d_obs, obs_b + (packed ? sizeof(float) * 2 * (size_t)n : 0), cudaMemcpyDeviceToHost, sm));
    } else if (obs) {
      pack_env_out_kernel<<<B, T, 0, sm>>>(s->q, s->qd, s->reward, s->done, d_obs, M.n_q, M.n_qd, n, ns, packed ? 1 : 0);
      CUDA_TRY(cudaMemcpyAsync(obs, d_obs, obs_b + (packed ? sizeof(float) * 2 * (size_t)n : 0), cudaMemcpyDeviceToHost, sm));
    }
    if (!packed) {
      if (rewards) CUDA_TRY(cudaMemcpyAsync(rewards, s->reward, sizeof(float) * n, cudaMemcpyDeviceToHost, sm));
      if (dones) CUDA_TRY(cudaMemcpyAsync(dones, s->done, sizeof(float) * n, cudaMemcpyDeviceToHost, sm));
    }
    return 0;
  };
  // Zero-copy: pinned (mapped) caller buffers and the specialised kernel -> the step kernel itself reads the actions
  // from host memory and writes observations / rewards / dones there (coalesced, staged through shared memory): one
  // launch, no staging copies.
  static const bool no_zero_copy = getenv("TDS_B200_NO_ZEROCOPY") != nullptr;
  if (direct && !s->phase_clk && !no_zero_copy) {
    void *da = nullptr, *dob = nullptr, *dr = nullptr, *dd = nullptr;
    bool ok;
    if ((++s->zc_calls & 63u) != 0 && s->zc_key[0] == actions && s->zc_key[1] == obs && s->zc_key[2] == rewards && s->zc_key[3] == dones) {
      ok = s->zc_ok;   // same buffers as the last call: the pointer queries (a microsecond each) are cached
      da = s->zc_dev[0]; dob = s->zc_dev[1]; dr = s->zc_dev[2]; dd = s->zc_dev[3];
    } else {
      ok = is_pinned(actions) && is_pinned(obs) && is_pinned(rewards) && is_pinned(dones);
      ok = ok && cudaHostGetDevicePointer(&da, (void*)actions, 0) == cudaSuccess;
      if (ok && obs) ok = cudaHostGetDevicePointer(&dob, obs, 0) == cudaSuccess;
      if (ok && rewards) ok = cudaHostGetDevicePointer(&dr, rewards, 0) == cudaSuccess;
      if (ok && dones) ok = cudaHostGetDevicePointer(&dd, dones, 0) == cudaSuccess;
      if (!ok) cudaGetLastError();
      s->zc_key[0] = actions; s->zc_key[1] = obs; s->zc_key[2] = rewards; s->zc_key[3] = dones;
      s->zc_dev[0] = da; s->zc_dev[1] = dob; s->zc_dev[2] = dr; s->zc_dev[3] = dd;
      s->zc_ok = ok;
    }
    if (ok) {
      s->io_act_aos = (const float*)da; s->io_obs_aos = (float*)dob; s->io_obs_tail = nullptr;
      rc = tds_b200_step_device(s, TDS_B200_MODE_FULL, 1, s->q, s->qd, s->act, s->q, s->qd, nullptr, dr ? (float*)dr : s->reward,
                                dd ? (float*)dd : s->done, nullptr, nullptr, sm);
      s->io_act_aos = nullptr; s->io_obs_aos = nullptr;
      if (rc) return rc;
      CUDA_TRY(cudaStreamSynchronize(sm));
      CUDA_TRY(cudaGetLastError());
      return 0;
    }
  }
  const void* key[4] = {actions, obs, rewards, dones};
  const bool same = s->g_key[0] == key[0] && s->g_key[1] == key[1] && s->g_key[2] == key[2] && s->g_key[3] == key[3];
  // the role-warp kernel reads its link table from ONE constant symbol per device: if another simulator took the symbol over
  // since the capture, the captured launch would run on that simulator's table - drop the graph, the eager path re-uploads
  if (s->g_exec && s->kernel == 3 && tds_stepr_table_owner(s->device) != s->table_token) drop_host_graph(s);
  if (same && s->g_exec) {
    CUDA_TRY(cudaGraphLaunch(s->g_exec, sm));
  } else if (same && s->g_seen >= 2 && !s->phase_clk && is_pinned(actions) && is_pinned(obs) && is_pinned(rewards) && is_pinned(dones)) {
    // third call with the same pinned buffers (the first two ran eagerly: lazy kernel attributes are set): capture
    cudaGraph_t g = nullptr;
    CUDA_TRY(cudaStreamBeginCapture(sm, cudaStreamCaptureModeThreadLocal));
    rc = enqueue();
    cudaError_t ce = cudaStreamEndCapture(sm, &g);
    if (rc || ce != cudaSuccess) {
      if (g) cudaGraphDestroy(g);
      cudaGetLastError();
      s->g_seen = -1000000;   // do not try again for this buffer set
      rc = enqueue();
      if (rc) return rc;
    } else {
      ce = cudaGraphInstantiate(&s->g_exec, g, 0);
      cudaGraphDestroy(g);
      if (ce != cudaSuccess) { s->g_exec = nullptr; set_err(std::string("cudaGraphInstantiate: ") + cudaGetErrorString(ce)); return (int)ce; }
      CUDA_TRY(cudaGraphLaunch(s->g_exec, sm));
    }
  } else {
    if (!same) { drop_host_graph(s); for (int k = 0; k < 4; ++k) s->g_key[k] = key[k]; }
    ++s->g_seen;
    rc = enqueue();
    if (rc) return rc;
  }
  CUDA_TRY(cudaStreamSynchronize(sm));
  CUDA_TRY(cudaGetLastError());
  return 0;
}

// ---- C-ABI v1 drop-in (src/utils/cuda_codegen.hpp:156-266) for the models ars_train_policy_cuda loads by name
// "cuda_model_" + env_name() (examples/ars/ars_train_policy_cuda.cpp:507): cuda_model_laikago and cuda_model_ant -------
static const double k_laikago_model[] = {
#include "generated/laikago_model.inc"
};
static const double k_ant_model[] = {
#include "generated/ant_model.inc"
};
struct V1Spec {
  const char* name;
  const double* model; int n_model;
  int in_dim, out_dim, written;       // written = n_q + n_qd + 7 * n_visuals + 1 (the rest of output_dim is never written)
  int n_q, n_act;
  double dt, init[TDS_MAX_ACT], kp, kd, max_force;
  int reward_kind;
};
// LaikagoContactSimulation: laikago_environment2.h:36-61, locomotion_contact_simulation.h:131-135 (51 -> 411)
static const V1Spec k_v1_laikago = {"cuda_model_laikago", k_laikago_model, (int)(sizeof(k_laikago_model) / sizeof(double)), 51, 411, 156, 18, 12,
                                    1e-3, {0.2, 0, -0.7, 0.2, 0, -0.7, 0.2, 0, -0.7, 0.2, 0, -0.7}, 100.0, 2.0, 50.0, 1};
// AntContactSimulation2: ant_environment2.h:28-70 (39 = q14|qd14|action8|kp,kd,max_force -> 155 = 28 + 14 links x 9 visuals + 1)
static const V1Spec k_v1_ant = {"cuda_model_ant", k_ant_model, (int)(sizeof(k_ant_model) / sizeof(double)), 39, 155, 92, 14, 8,
                                0.01, {0.0, -0.5, 0.0, -0.5, 0.0, -0.5, 0.0, -0.5}, 15.0, 0.3, 3.0, 3};
struct V1Instance {
  tds_b200_sim* sim = nullptr;
  double *dev_in = nullptr, *dev_out = nullptr;
  int n = 0;
  std::mutex mu;
};
static V1Instance g_v1_laikago, g_v1_ant;

static void v1_fail(const V1Spec& S, const char* what) {
  // the reference prints and exits on allocation failure (cuda_codegen.hpp:201-208)
  fprintf(stderr, "%s (tds_b200): %s: %s\n", S.name, what, g_err.c_str());
  exit(1);
}

static void v1_release(V1Instance& I) {
  if (I.sim) tds_b200_destroy(I.sim);
  I.sim = nullptr;
  cudaFree(I.dev_in); cudaFree(I.dev_out);
  I.dev_in = I.dev_out = nullptr;
  I.n = 0;
}

static void v1_allocate(V1Instance& I, const V1Spec& S, int num_total_threads) {
  std::lock_guard<std::mutex> lk(I.mu);
  v1_release(I);
  int dev = 0;
  cudaGetDevice(&dev);
  I.sim = tds_b200_create(S.model, S.n_model, num_total_threads, dev);
  if (!I.sim) v1_fail(S, "allocate");
  const double g[3] = {0, 0, -9.81};
  tds_b200_set_params(I.sim, S.dt, g, 1.0, 0.0, 0.2, 1e-5, 1, 1);
  tds_b200_set_env(I.sim, S.n_act, S.init, 6, S.kp, S.kd, S.max_force, 0.4, S.reward_kind);
  I.n = num_total_threads;
  if (cudaMalloc((void**)&I.dev_in, sizeof(double) * (size_t)num_total_threads * S.in_dim) != cudaSuccess ||
      cudaMalloc((void**)&I.dev_out, sizeof(double) * (size_t)num_total_threads * S.written) != cudaSuccess) {
    set_err("cudaMalloc failed");
    v1_fail(S, "allocate");
  }
}

static void v1_forward_zero(V1Instance& I, const V1Spec& S, int num_total_threads, double* output, const double* input) {
  std::lock_guard<std::mutex> lk(I.mu);
  if (!I.sim || num_total_threads > I.n) { set_err("forward_zero called before allocate (or with more threads)"); v1_fail(S, "forward_zero"); }
  tds_b200_sim* s = I.sim;
  const int n = num_total_threads, ns = s->ns;
  cudaStream_t sm = s->stream;
  const int T = 128, B = (n + T - 1) / T;
  const int saved_n = s->n;
  s->n = n;
  cudaMemcpyAsync(I.dev_in, input, sizeof(double) * (size_t)n * S.in_dim, cudaMemcpyHostToDevice, sm);
  aos_to_soa_kernel<double><<<B, T, 0, sm>>>(I.dev_in, S.in_dim, 0, s->q, S.n_q, n, ns);
  aos_to_soa_kernel<double><<<B, T, 0, sm>>>(I.dev_in, S.in_dim, S.n_q, s->qd, S.n_q, n, ns);
  aos_to_soa_kernel<double><<<B, T, 0, sm>>>(I.dev_in, S.in_dim, 2 * S.n_q, s->act, S.n_act, n, ns);
  // kp, kd, max_force travel in the input vector (locomotion_contact_simulation.h:164-166); the v1 ABI is
  // called with one value for the whole batch (ars_vectorized_environment.h:223-236): read env 0's.
  const int v0 = 2 * S.n_q + S.n_act;
  s->E.kp = (float)input[v0]; s->E.kd = (float)input[v0 + 1]; s->E.max_force = (float)input[v0 + 2];
  int rc = tds_b200_step_device(s, TDS_B200_MODE_FULL, 1, s->q, s->qd, s->act, s->q, s->qd, nullptr, nullptr, nullptr,
                                nullptr, s->link_xf, sm);
  if (rc) v1_fail(S, "step");
  pack_v1_output_kernel<<<B, T, 0, sm>>>(s->vis, s->q, s->qd, s->link_xf, I.dev_out, S.written, n, ns, s->dm[0].floating);
  // entries >= written are never written by the reference either (they keep the caller's values)
  cudaMemcpy2DAsync(output, sizeof(double) * S.out_dim, I.dev_out, sizeof(double) * S.written, sizeof(double) * S.written, n,
                    cudaMemcpyDeviceToHost, sm);
  cudaError_t e = cudaStreamSynchronize(sm);
  s->n = saved_n;
  if (e != cudaSuccess) { set_err(cudaGetErrorString(e)); v1_fail(S, "forward_zero"); }
}

#define TDS_V1_SYMBOLS(model, inst, spec)                                                                              \
  CudaFunctionMetaData model##_forward_zero_meta(void) {                                                               \
    CudaFunctionMetaData d; d.output_dim = spec.out_dim; d.input_dim = spec.in_dim; d.global_dim = 0; return d;        \
  }                                                                                                                    \
  void model##_forward_zero_allocate(int num_total_threads) { v1_allocate(inst, spec, num_total_threads); }            \
  void model##_forward_zero_deallocate(void) { std::lock_guard<std::mutex> lk(inst.mu); v1_release(inst); }            \
  void model##_forward_zero(int num_total_threads, int num_blocks, int num_threads_per_block, double* output,          \
                            const double* input) {                                                                     \
    (void)num_blocks; (void)num_threads_per_block;                                                                     \
    v1_forward_zero(inst, spec, num_total_threads, output, input);                                                     \
  }
TDS_V1_SYMBOLS(cuda_model_laikago, g_v1_laikago, k_v1_laikago)
TDS_V1_SYMBOLS(cuda_model_ant, g_v1_ant, k_v1_ant)
static const int k_laikago_in = 51, k_laikago_out = 411;

// ---- C-ABI v2 (src/utils/cuda/cuda_codegen.hpp:32-231, loaded by tds::CudaLibrary / CudaModel / CudaFunction,
// src/utils/cuda/cuda_{library,model,function}.hpp): model_info + <model>_forward_zero{,_meta,_allocate,_deallocate,
// _send_local,_send_global}.  The model is exported as "b200_laikago" (the v1 symbols keep the name cuda_model_laikago:
// the two generations use the same symbol names with different meta structs, so they cannot share a model name).
// <model>_jacobian: b200_laikago_jacobian below (forward-mode dual numbers through the step kernel).
static std::vector<double> g_v2_local;   // thread-local inputs as last sent ([n][51], host)
static int g_v2_sent = 0;

void model_info(char const* const** names, int* count) {
  static const char* k_names[1] = {"b200_laikago"};
  *names = k_names;
  *count = 1;
}

CudaFunctionMetaDataV2 b200_laikago_forward_zero_meta(void) {
  CudaFunctionMetaDataV2 d;
  d.output_dim = k_laikago_out; d.local_input_dim = k_laikago_in; d.global_input_dim = 0; d.accumulated_output = false;
  return d;
}

void b200_laikago_forward_zero_allocate(int num_total_threads) {
  cuda_model_laikago_forward_zero_allocate(num_total_threads);
  g_v2_local.assign((size_t)num_total_threads * k_laikago_in, 0.0);
  g_v2_sent = 0;
}

void b200_laikago_forward_zero_deallocate(void) {
  cuda_model_laikago_forward_zero_deallocate();
  g_v2_local.clear(); g_v2_local.shrink_to_fit();
  g_v2_sent = 0;
}

bool b200_laikago_forward_zero_send_local(int num_total_threads, const double* input) {
  if (!input || (size_t)num_total_threads * k_laikago_in > g_v2_local.size()) {
    fprintf(stderr, "Error while sending thread-local input data to GPU: %d threads exceed the allocation.\n", num_total_threads);
    return false;
  }
  memcpy(g_v2_local.data(), input, sizeof(double) * (size_t)num_total_threads * k_laikago_in);
  g_v2_sent = num_total_threads;
  return true;
}

bool b200_laikago_forward_zero_send_global(const double* input) { (void)input; return true; }   // global_input_dim = 0

void b200_laikago_forward_zero(int num_total_threads, int num_blocks, int num_threads_per_block, double* output) {
  if (num_total_threads > g_v2_sent) { fprintf(stderr, "b200_laikago_forward_zero: launch before send_local\n"); exit(1); }
  cuda_model_laikago_forward_zero(num_total_threads, num_blocks, num_threads_per_block, output, g_v2_local.data());
}

// <model>_jacobian of the v2 generation (CudaModelSourceGen::jacobian_source, src/utils/cuda/cuda_codegen.hpp:303-426;
// loaded by tds::CudaModel as the function named "<model>_jacobian", src/utils/cuda/cuda_model.hpp:14-25): dense rows
// (output_i, input_i) in row-major order per thread.  Output sparsity (set_jac_output_sparsity, :283-288): the 36 state
// rows q' | qd' of the 411 outputs; all 51 local inputs (q | qd | action | kp, kd, max_force) as columns; no accumulation.
static V1Instance g_v2_jac;
static std::vector<double> g_v2_jac_local;
static int g_v2_jac_sent = 0;
static const int k_jac_rows = 36, k_jac_cols = 51;

CudaFunctionMetaDataV2 b200_laikago_jacobian_meta(void) {
  CudaFunctionMetaDataV2 d;
  d.output_dim = k_jac_rows * k_jac_cols; d.local_input_dim = k_laikago_in; d.global_input_dim = 0; d.accumulated_output = false;
  return d;
}
void b200_laikago_jacobian_allocate(int num_total_threads) {
  v1_allocate(g_v2_jac, k_v1_laikago, num_total_threads);
  g_v2_jac_local.assign((size_t)num_total_threads * k_laikago_in, 0.0);
  g_v2_jac_sent = 0;
}
void b200_laikago_jacobian_deallocate(void) {
  { std::lock_guard<std::mutex> lk(g_v2_jac.mu); v1_release(g_v2_jac); }
  g_v2_jac_local.clear(); g_v2_jac_local.shrink_to_fit();
  g_v2_jac_sent = 0;
}
bool b200_laikago_jacobian_send_local(int num_total_threads, const double* input) {
  if (!input || (size_t)num_total_threads * k_laikago_in > g_v2_jac_local.size()) {
    fprintf(stderr, "Error while sending thread-local input data to GPU: %d threads exceed the allocation.\n", num_total_threads);
    return false;
  }
  memcpy(g_v2_jac_local.data(), input, sizeof(double) * (size_t)num_total_threads * k_laikago_in);
  g_v2_jac_sent = num_total_threads;
  return true;
}
bool b200_laikago_jacobian_send_global(const double* input) { (void)input; return true; }
void b200_laikago_jacobian(int num_total_threads, int num_blocks, int num_threads_per_block, double* output) {
  (void)num_blocks; (void)num_threads_per_block;
  std::lock_guard<std::mutex> lk(g_v2_jac.mu);
  if (!g_v2_jac.sim || num_total_threads > g_v2_jac_sent) { fprintf(stderr, "b200_laikago_jacobian: launch before allocate / send_local\n"); exit(1); }
  tds_b200_sim* s = g_v2_jac.sim;
  const int n = num_total_threads;
  std::vector<double> q((size_t)n * 18), qd((size_t)n * 18), act((size_t)n * 12);
  for (int e = 0; e < n; ++e) {
    const double* x = g_v2_jac_local.data() + (size_t)e * k_laikago_in;
    memcpy(&q[(size_t)e * 18], x, 18 * sizeof(double)); memcpy(&qd[(size_t)e * 18], x + 18, 18 * sizeof(double));
    memcpy(&act[(size_t)e * 12], x + 36, 12 * sizeof(double));
  }
  s->E.kp = (float)g_v2_jac_local[48]; s->E.kd = (float)g_v2_jac_local[49]; s->E.max_force = (float)g_v2_jac_local[50];
  const int saved_n = s->n;
  s->n = n;
  const int rc = tds_b200_step_jacobian_host(s, TDS_B200_MODE_FULL, 1, q.data(), qd.data(), act.data(), output);
  s->n = saved_n;
  if (rc) { fprintf(stderr, "b200_laikago_jacobian: %s\n", g_err.c_str()); exit(1); }
}

}  // extern "C"
