// TEST INFRASTRUCTURE - NOT PRODUCT CODE, never loaded by the package.
//
// The table-driven tree kernels - the step body tiny-differentiable-simulator_b200/csrc/tds_team_step.cuh under its two thread
// mappings, LaneTeam (tds_stept.cu: 8 environments x 4 lanes per warp) and RoleWarps (tds_stepr.cu: 32 environments x 4 role
// warps per CTA) - compiled FOR THE HOST, over the partition and tables the library builds (tds_team.h).
//
// Every thread of a tile is a coroutine with its own stack; all of them are alive together but only one runs at a time.  The
// baton passes at every barrier and warp collective, to the lowest (ascending order) or highest (descending order) thread index
// that may run.  A run is therefore deterministic, and a missing or misplaced barrier shows deterministically: one of the two
// orders lets a reader see the value before its writer produced it.  Emulated primitives:
//   __syncthreads / __syncthreads_or   barrier of every thread of the tile, with an OR-reduction (RoleWarps)
//   __syncwarp()                       barrier of the 32 threads of the warp = the tile (LaneTeam)
//   __syncwarp(tmask)                  barrier of the 4 threads of one team (LaneTeam)
//   __shfl_xor_sync / __shfl_sync      team collectives: write a per-thread slot, team barrier, read the partner's slot, team
//                                      barrier; a full-mask __shfl_sync (RoleWarps::role(): the warp index) returns its argument
//   __ldg, __ffsll                     plain load, __builtin_ffsll;  c_team: an ordinary array filled from tds_build_team's table
// A barrier that can never complete (threads of a tile waiting at different barriers, or some of them finished) is found when
// no thread may run, and a tile that is still passing barriers after 10 s is abandoned: either way the call returns a negative
// code instead of hanging.  Shared memory is one static array reused by the tiles one after another (SMEM = true) or one global
// block per tile (SMEM = false); both are filled with NaN bytes before use, so a read of a word nobody wrote poisons the result.
//   g++ -std=c++17 -O1 -shared -fPIC -I<csrc> -I<include> -I/usr/local/cuda/include tests/cpp/team_host.cpp -o tests/cpp/_team_host.so
#include <cuda_runtime.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <ucontext.h>

#include <chrono>
#include <vector>

#define TDS_B200_EXACT_RCP 1
#define TDS_TEAM_KERNEL_ONLY 1

namespace emu {
struct Dim { unsigned x, y, z; };
Dim tIdx, bIdx, bDim;

enum { RUNNABLE = 0, WAITING = 1, DONE = 2 };
constexpr int MAXT = 128;            // threads of the largest tile (RoleWarps: 4 warps)
constexpr size_t STACK = 1 << 20;    // per coroutine (the kernel's parameters alone are tens of KB)
struct Co { ucontext_t ctx; int state, bar, result; unsigned tid; };
Co co[MAXT];
char* stacks = nullptr;
ucontext_t main_ctx;
int n_co = 0, cur = 0, descending = 0, team_barriers = 0, force_or = 0, err = 0;
unsigned block = 0;
struct Bar { int arrived, acc; };
Bar bars[1 + MAXT / 4];               // 0: the tile; 1 + t: team t (LaneTeam)
unsigned long long slot[MAXT];         // shuffle exchange, one per thread
void (*body)() = nullptr;

// arrive at barrier `key` with `members` threads, hand the baton back to the scheduler, return the OR of the predicates
inline int arrive(int key, int members, int pred) {
  Bar& b = bars[key];
  b.acc |= pred ? 1 : 0;
  co[cur].state = WAITING; co[cur].bar = key;
  if (++b.arrived == members) {
    for (int i = 0; i < n_co; ++i)
      if (co[i].state == WAITING && co[i].bar == key) { co[i].state = RUNNABLE; co[i].result = b.acc; }
    b.arrived = 0; b.acc = 0;
  }
  swapcontext(&co[cur].ctx, &main_ctx);
  return co[cur].result;
}
inline int tile_sync(int pred) { return arrive(0, n_co, pred); }
inline unsigned team_mask() { return 0xFu << ((co[cur].tid & 31) & ~3u); }
inline void team_sync(unsigned mask) {
  if (!team_barriers || mask != team_mask()) err = err ? err : -12;   // a mask that is not the caller's team
  arrive(1 + (int)((co[cur].tid & 31) >> 2), 4, 0);
}
template <typename T> T team_exchange(unsigned mask, T v, int src_lane) {
  static_assert(sizeof(T) <= sizeof(unsigned long long), "shuffle of a wider type");
  memcpy(&slot[cur], &v, sizeof(T));
  team_sync(mask);
  T r;
  memcpy(&r, &slot[src_lane & 31], sizeof(T));   // (LaneTeam: thread index = lane)
  team_sync(mask);
  return r;
}

void entry(int i) {
  body();
  co[i].state = DONE;
}   // returns to main_ctx through uc_link

// Runs `body` on threads tids[0..n) of block `blk`; returns 0, or -10 (a barrier no thread can complete), -11 (10 s timeout),
// -12 (a collective with a mask other than the caller's team).
int run_tile(const unsigned* tids, int n, unsigned blk) {
  if (!stacks) stacks = (char*)malloc(STACK * MAXT);   // untouched pages stay uncommitted
  n_co = n; block = blk; err = 0;
  memset(bars, 0, sizeof(bars));
  for (int i = 0; i < n; ++i) {
    co[i].state = RUNNABLE; co[i].tid = tids[i]; co[i].bar = -1; co[i].result = 0;
    getcontext(&co[i].ctx);
    co[i].ctx.uc_stack.ss_sp = stacks + (size_t)i * STACK;
    co[i].ctx.uc_stack.ss_size = STACK;
    co[i].ctx.uc_link = &main_ctx;
    makecontext(&co[i].ctx, (void (*)())entry, 1, i);
  }
  const auto t0 = std::chrono::steady_clock::now();
  for (long sw = 0;; ++sw) {
    int next = -1;
    if (!descending) { for (int i = 0; i < n; ++i) if (co[i].state == RUNNABLE) { next = i; break; } }
    else { for (int i = n - 1; i >= 0; --i) if (co[i].state == RUNNABLE) { next = i; break; } }
    if (next < 0) {
      for (int i = 0; i < n; ++i) if (co[i].state != DONE) return -10;
      return err;
    }
    if ((sw & 1023) == 1023 && std::chrono::steady_clock::now() - t0 > std::chrono::seconds(10)) return -11;
    cur = next;
    tIdx = {co[next].tid, 0, 0};
    bIdx = {blk, 0, 0};
    swapcontext(&main_ctx, &co[next].ctx);
  }
}
}  // namespace emu

#define threadIdx emu::tIdx
#define blockIdx emu::bIdx
#define blockDim emu::bDim
#define __syncthreads() ((void)emu::tile_sync(0))
#define __syncthreads_or(p) (emu::tile_sync((p) ? 1 : 0) | emu::force_or)
#define clock64() (0LL)
static inline void __syncwarp(unsigned mask = 0xffffffffu) {
  if (mask == 0xffffffffu) emu::tile_sync(0);   // LaneTeam: the warp is the tile
  else emu::team_sync(mask);
}
template <typename T> static inline T __shfl_xor_sync(unsigned mask, T v, int lane_mask) {
  return emu::team_exchange(mask, v, (int)(emu::co[emu::cur].tid & 31) ^ lane_mask);
}
template <typename T> static inline T __shfl_sync(unsigned mask, T v, int src_lane) {
  if (mask == 0xffffffffu) return v;   // warp-uniform argument (RoleWarps::role)
  return emu::team_exchange(mask, v, src_lane);
}
static inline int __ffsll(long long x) { return __builtin_ffsll(x); }
template <typename T> static inline T __ldg(const T* p) { return *p; }
#undef __shared__
#define __shared__
#undef __constant__
#define __constant__
#undef __grid_constant__
#define __grid_constant__
#undef __global__
#define __global__
#undef __launch_bounds__
#define __launch_bounds__(...)
#define smem_raw emu_smem_raw

#include "../../tiny-differentiable-simulator_b200/csrc/tds_stept.cu"
#include "../../tiny-differentiable-simulator_b200/csrc/tds_stepr.cu"

namespace tdsteam { alignas(16) char emu_smem_raw[32 << 20]; }   // the tile's shared memory (block-scope extern in the kernel)

namespace {
using tdsteam::LaneTeam;
using tdsteam::RoleWarps;

struct Call {
  TeamModel TM; DevModel M; SimParams P; EnvParams E; StepIO io;
  const TeamLink* tl; int mode, use_pd; char* gscratch;
};
Call* g_call = nullptr;

template <class Map, typename RA, typename RC, typename RS, bool SMEM> void body() {
  const Call& c = *g_call;
  tdsteam::tds_team_step_kernel<Map, RA, RC, RS, SMEM>(c.TM, c.tl, c.M, c.P, c.E, c.io, c.mode, c.use_pd, c.gscratch);
}

// lane_by_lane (RoleWarps only): the 4 role threads of one environment at a time instead of the tile's 128 threads
template <class Map, typename RA, typename RC, typename RS, bool SMEM> int run(Call& c, int lane_by_lane) {
  emu::body = body<Map, RA, RC, RS, SMEM>;
  emu::team_barriers = Map::ROLE_WARPS ? 0 : 1;
  emu::bDim = {(unsigned)Map::THREADS, 1, 1};
  const size_t tb = Map::tile_bytes(c.TM);
  const int tiles = (c.io.n + Map::STM - 1) / Map::STM;
  std::vector<char> gs;
  if (SMEM) { if (tb > sizeof(tdsteam::emu_smem_raw)) return -4; }
  else { gs.assign(tb * tiles, (char)0xff); c.gscratch = gs.data(); }
  g_call = &c;
  unsigned tids[emu::MAXT];
  for (int t = 0; t < tiles; ++t) {
    if (SMEM) memset(tdsteam::emu_smem_raw, 0xff, tb);
    if (Map::ROLE_WARPS && lane_by_lane) {
      for (int lane = 0; lane < 32 && t * 32 + lane < c.io.n; ++lane) {
        for (int r = 0; r < TDS_TEAM_T; ++r) tids[r] = (unsigned)(r * 32 + lane);
        if (int rc = emu::run_tile(tids, TDS_TEAM_T, (unsigned)t)) return rc;
      }
    } else {
      for (int i = 0; i < Map::THREADS; ++i) tids[i] = (unsigned)i;
      if (int rc = emu::run_tile(tids, Map::THREADS, (unsigned)t)) return rc;
    }
  }
  return 0;
}

template <class Map, bool SMEM> int run_prec(Call& c, int precision, int lane_by_lane) {
  if (precision == 0) return run<Map, float, double, float, SMEM>(c, lane_by_lane);
  if (precision == 1) return run<Map, double, double, double, SMEM>(c, lane_by_lane);
  return run<Map, float, float, float, SMEM>(c, lane_by_lane);
}

const int kSizes[3][3] = {{4, 8, 4}, {8, 8, 8}, {4, 4, 4}};   // sizeof(RA, RC, RS) per precision (tds_capi.cu)

// DevModel, EnvParams and TeamModel + table as the library builds them (tds_b200_create, tds_b200_set_env, rebuild_team).
// Returns the model's error code (-30: fewer actuated links than n_act); tds_build_team's code in *team_rc.
int setup(const double* model, int n_model, const double* env, DevModel* D, EnvParams* E, TeamModel* TM, std::vector<TeamLink>* table,
          int* team_rc) {
  int rc = tds_build_dev_model(model, n_model, D);
  if (rc) return rc;
  memset(E, 0, sizeof(*E));
  if (env) {   // n_act, start_link, kp, kd, max_force, action_limit, reward_kind, auto_reset, poses[n_act], reset_q[n_q]
    E->n_act = (int)env[0]; E->start_link = (int)env[1];
    E->kp = (float)env[2]; E->kd = (float)env[3]; E->max_force = (float)env[4]; E->action_limit = (float)env[5];
    E->reward_kind = (int)env[6]; E->auto_reset = (int)env[7];
    int k = 0;
    for (int i = D->floating ? 0 : E->start_link; i < D->n_links && k < E->n_act; ++i) {
      if (D->flags[i] & TDS_LF_FIXED) continue;
      E->act_link[k] = i; E->initial_poses[k] = (float)env[8 + k]; ++k;
    }
    if (k != E->n_act) return -30;
    for (int j = 0; j < D->n_q; ++j) E->reset_q[j] = (float)env[8 + E->n_act + j];
  }
  *team_rc = tds_build_team(D, E, TM, table);
  return 0;
}
}  // namespace

extern "C" {

// map 0 LaneTeam / 1 RoleWarps; precision 0 mixed / 1 fp64 / 2 fp32; smem 1: the shared-memory instance, 0: global scratch.
// params: dt, g[3], friction, restitution, erp, cfm, pgs_iterations, keep_all (10 doubles); env as in setup() or null.
// flags: bit 0 force_or (every __syncthreads_or is true, as when another lane of the tile has a contact), bit 1 lane_by_lane
// (RoleWarps), bit 2 descending baton order.  Host layout [n][dim]; outputs may be null; contact_dist [n][n_cand],
// link_xf [n][n_links * 12].  Returns n_cand, or < 0: -100 + the model's error code, -3 tds_build_team did not decompose the
// model, -4 tile too large for the emulated shared memory, -10 / -11 / -12 see emu::run_tile.
int tdsemu_team_step(const double* model, int n_model, const double* params, const double* env, int map, int precision, int smem,
                     int mode, int use_pd, int flags, int n, const double* q, const double* qd, const double* tau, double* q_out,
                     double* qd_out, double* qdd_out, double* reward, double* done, double* contact_dist, double* link_xf) {
  Call* c = new Call;
  std::vector<TeamLink> table;
  memset(c, 0, sizeof(*c));
  int team_rc = 0;
  int rc = setup(model, n_model, env, &c->M, &c->E, &c->TM, &table, &team_rc);
  if (rc || team_rc) { delete c; return rc ? -100 + rc : -3; }
  tds_build_layout(&c->M, kSizes[precision][0], kSizes[precision][1], kSizes[precision][2], -1);
  tds_build_layout_w(&c->M, kSizes[precision][0], kSizes[precision][1], kSizes[precision][2], -1);
  tds_build_team_layout(&c->TM, kSizes[precision][0], kSizes[precision][1], kSizes[precision][2]);
  memcpy(tdsteam::c_team, table.data(), sizeof(TeamLink) * TDS_TEAM_T * TDS_TEAM_MAXK);
  c->tl = table.data();
  SimParams& P = c->P;
  P.dt = params[0]; P.inv_dt = 1.0 / params[0];
  for (int k = 0; k < 3; ++k) P.gravity[k] = params[1 + k];
  P.friction = params[4]; P.restitution = params[5]; P.erp = params[6]; P.cfm = params[7];
  P.pgs_iterations = (int)params[8]; P.keep_all_points = (int)params[9];
  const DevModel& D = c->M;
  const int ns = (n + 31) & ~31, n_q = D.n_q, n_qd = D.n_qd, n_cand = c->TM.n_cand, n_links = D.n_links;
  const int n_tau = n_qd - (D.floating ? 6 : 0), n_in = use_pd ? c->E.n_act : n_tau;
  auto rows = [](int r) { return (size_t)(r > 0 ? r : 1); };
  std::vector<float> sq(rows(n_q) * ns), sqd(rows(n_qd) * ns), st(rows(n_in) * ns, 0.f), oq(sq.size()), oqd(sqd.size()),
      oqdd(sqd.size()), orew(ns), odone(ns), ocd(rows(n_cand) * ns), oxf(rows(n_links * 12) * ns);
  for (int e = 0; e < n; ++e) {
    for (int k = 0; k < n_q; ++k) sq[(size_t)k * ns + e] = (float)q[(size_t)e * n_q + k];
    for (int k = 0; k < n_qd; ++k) sqd[(size_t)k * ns + e] = (float)qd[(size_t)e * n_qd + k];
    if (tau) for (int k = 0; k < n_in; ++k) st[(size_t)k * ns + e] = (float)tau[(size_t)e * n_in + k];
  }
  StepIO& io = c->io;
  io.q_in = sq.data(); io.qd_in = sqd.data(); io.tau_in = (tau || use_pd) ? st.data() : nullptr;
  io.q_out = oq.data(); io.qd_out = oqd.data(); io.qdd_out = oqdd.data();
  io.reward = orew.data(); io.done = odone.data();
  io.contact_dist = contact_dist ? ocd.data() : nullptr;
  io.link_xf = link_xf ? oxf.data() : nullptr;
  io.n = n; io.n_stride = ns;
  c->mode = mode; c->use_pd = use_pd;
  emu::force_or = flags & 1;
  emu::descending = (flags >> 2) & 1;
  const int lane_by_lane = (flags >> 1) & 1;
  if (map == 0) rc = smem ? run_prec<LaneTeam, true>(*c, precision, 0) : run_prec<LaneTeam, false>(*c, precision, 0);
  else rc = smem ? run_prec<RoleWarps, true>(*c, precision, lane_by_lane) : run_prec<RoleWarps, false>(*c, precision, lane_by_lane);
  if (rc == 0)
    for (int e = 0; e < n; ++e) {
      if (q_out) for (int k = 0; k < n_q; ++k) q_out[(size_t)e * n_q + k] = oq[(size_t)k * ns + e];
      if (qd_out) for (int k = 0; k < n_qd; ++k) qd_out[(size_t)e * n_qd + k] = oqd[(size_t)k * ns + e];
      if (qdd_out) for (int k = 0; k < n_qd; ++k) qdd_out[(size_t)e * n_qd + k] = oqdd[(size_t)k * ns + e];
      if (reward) reward[e] = orew[e];
      if (done) done[e] = odone[e];
      if (contact_dist) for (int k = 0; k < n_cand; ++k) contact_dist[(size_t)e * n_cand + k] = ocd[(size_t)k * ns + e];
      if (link_xf) for (int k = 0; k < n_links * 12; ++k) link_xf[(size_t)e * n_links * 12 + k] = oxf[(size_t)k * ns + e];
    }
  delete c;
  return rc ? rc : n_cand;
}

// Summary of the partition tds_build_team makes of a model (env as for tdsemu_team_step, or null).  out (TDSEMU_INFO doubles):
//  [0] tds_build_team's return code  [1] n_trunk  [2..5] n_loc  [6..9] n_od  [10] n_att  [11] n_acc  [12] n_xw_team
//  [13] n_xw_lane  [14] n_cand  [15] trunk-internal accumulator slots  [16] own-internal accumulator slots (most of one role)
//  [17] kmax  [18] floating  [19] subtrees on a fixed base (dropped contributions)  [20..22] LaneTeam tile bytes (mixed, fp64,
//  fp32)  [23..25] RoleWarps tile bytes  [26..29] subtrees per role  [30..77] cand_owner.  Returns the model's error code or 0.
int tdsemu_team_info(const double* model, int n_model, const double* env, double* out) {
  DevModel* D = new DevModel;
  EnvParams E;
  TeamModel TM;
  std::vector<TeamLink> table;
  memset(out, 0, sizeof(double) * 78);
  int rc = 0;
  const int mrc = setup(model, n_model, env, D, &E, &TM, &table, &rc);
  if (mrc) { delete D; return mrc; }
  out[0] = rc;
  if (rc == 0) {
    out[1] = TM.n_trunk;
    for (int r = 0; r < 4; ++r) { out[2 + r] = TM.n_loc[r]; out[6 + r] = TM.n_od[r]; }
    out[10] = TM.n_att; out[11] = TM.n_acc; out[12] = TM.n_xw_team; out[13] = TM.n_xw_lane; out[14] = TM.n_cand;
    std::vector<int> trunk_int, own_int[4];
    int dropped = 0;
    for (int r = 0; r < 4; ++r) {
      int roots = 0;
      for (int k = 0; k < TM.n_loc[r]; ++k) {
        const TeamLink& L = table[(size_t)r * TDS_TEAM_MAXK + k];
        if (k >= TM.n_trunk && (L.flags & TDS_TF_PARENT_TRUNK)) { ++roots; if (L.par_slot < 0) ++dropped; }
        if (L.par_slot < TM.n_att) continue;
        std::vector<int>& v = k < TM.n_trunk ? trunk_int : own_int[r];
        if (std::find(v.begin(), v.end(), L.par_slot) == v.end()) v.push_back(L.par_slot);
      }
      out[26 + r] = roots;
    }
    out[15] = (double)trunk_int.size();
    for (int r = 0; r < 4; ++r) out[16] = std::max(out[16], (double)own_int[r].size());
    out[17] = TM.kmax; out[18] = TM.floating; out[19] = dropped;
    for (int p = 0; p < 3; ++p) {
      TeamModel t = TM;
      tds_build_team_layout(&t, kSizes[p][0], kSizes[p][1], kSizes[p][2]);
      out[20 + p] = (double)LaneTeam::tile_bytes(t);
      out[23 + p] = (double)RoleWarps::tile_bytes(t);
    }
    for (int g = 0; g < TM.n_cand; ++g) out[30 + g] = TM.cand_owner[g];
  }
  delete D;
  return 0;
}

}  // extern "C"
