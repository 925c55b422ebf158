"""The table-driven tree kernels - the step body csrc/tds_team_step.cuh under its two thread mappings, lane teams
(csrc/tds_stept.cu) and role warps (csrc/tds_stepr.cu) - executed on the CPU by compiling their SOURCE for the host
(tests/cpp/team_host.cpp), over the partition tds_build_team makes of the fixture models, of random trees and of hand-made
trees that reach the partition's rarer branches: a trunk grown past the root, several subtrees on one role, roles that own
nothing, trunk-internal and own-internal accumulators, subtrees on a fixed base, contact rows of several owners, and the
capacity edges TDS_TEAM_MAXK / TDS_TEAM_MAXC.  These kernels serve every tree model without a compiled instance (the
humanoid, and any robot a user compiles from a URDF).  The threads of a tile take turns in a fixed order at every barrier, so
a missing barrier changes the result deterministically (ascending against descending order).  tests/test_team_kernels_gpu.py
takes the same trees and states through the library on the GPU."""
import functools
import zlib

import numpy as np
import pytest

import emu
import emu_team
import tds_b200.envs as envs
from oracle import port
from tds_b200.model import compile_urdf, fixture_path, load_model
from test_model_compiler import PLANE, _random_urdf

N = 40                 # environments per (tree, variant): two role-warp tiles (the second ragged), five lane-team tiles
TOL64 = 2e-7           # fp64 arithmetic against the fp64 oracle (DESIGN.md section 2)
C_MIXED = 6.0          # mixed / fp32 arithmetic: err_tree <= C_MIXED * err_world + 1e-6 (see test_mixed_and_fp32_against_the_world_kernel)
# (tree, precision, mode) -> bound on err_tree where the ratio exceeds 10, each explained where it is used
MIXED_KNOWN = {("hand-nonadjacent_trunk_child", 0, port.MODE_NOCONTACT): 2e-5}
RANDOM_SEEDS = range(40)
MODES = (port.MODE_FD, port.MODE_NOCONTACT, port.MODE_FULL)

# flat model layout (include/tds_b200_model.h)
H, BASE, LINK = 16, 13, 34
L_PARENT, L_JTYPE, L_QIDX, L_QDIDX, L_XT_T = 0, 1, 2, 3, 16
J_FIXED = -1


def rel_err(a, ref):
    return float(np.max(np.abs(a - ref) / np.maximum(1.0, np.abs(ref)))) if ref.size else 0.0


def _link(model, i, field):
    return model[H + BASE + i * LINK + field]


# ---- hand-made trees --------------------------------------------------------------------------------------------------------
def _tree_urdf(parents, seed, joints=None, geoms=None, reach=0.25):
    """URDF of a tree: link 0 is the base, parents[i - 1] the parent of link i.  joints: {link: type} (default: revolute about a
    random axis); geoms: {link: "s" | "c" | "cc"} spheres / capsules.  Masses, inertias, origins and axes drawn from `seed`."""
    rng = np.random.default_rng(seed)
    joints, geoms = joints or {}, geoms or {}
    v3 = lambda lo, hi: " ".join("%.6g" % x for x in rng.uniform(lo, hi, 3))
    parts = ['<?xml version="1.0"?>', '<robot name="tree">']
    for i in range(len(parents) + 1):
        ixx, iyy, izz = rng.uniform(5e-3, 0.1, 3)
        col = ""
        for g in geoms.get(i, ""):
            geo = (f'<sphere radius="{rng.uniform(0.03, 0.08):.4g}"/>' if g == "s" else
                   f'<capsule radius="{rng.uniform(0.02, 0.05):.4g}" length="{rng.uniform(0.08, 0.2):.4g}"/>')
            col += f'<collision><origin xyz="{v3(-0.05, 0.05)}" rpy="{v3(-1, 1)}"/><geometry>{geo}</geometry></collision>'
        parts.append(f'<link name="l{i}"><inertial><origin xyz="{v3(-0.05, 0.05)}" rpy="{v3(-0.5, 0.5)}"/>'
                     f'<mass value="{rng.uniform(0.3, 3.0):.6g}"/><inertia ixx="{ixx:.6g}" iyy="{iyy:.6g}" izz="{izz:.6g}" ixy="0" ixz="0" '
                     f'iyz="0"/></inertial>{col}</link>')
    axes = ["1 0 0", "0 1 0", "0 0 1", "0 -1 0", "0.6 0 0.8", "0.3 -0.4 0.5"]
    for i, p in enumerate(parents, start=1):
        jt = joints.get(i, "revolute")
        axis = "" if jt == "fixed" else f'<axis xyz="{axes[rng.integers(0, len(axes))]}"/>'
        lim = '<limit lower="-1" upper="1" effort="10" velocity="10"/>' if jt in ("revolute", "prismatic") else ""
        parts.append(f'<joint name="j{i}" type="{jt}"><parent link="l{p}"/><child link="l{i}"/>'
                     f'<origin xyz="{v3(-reach, reach)}" rpy="{v3(-1, 1)}"/>{axis}{lim}</joint>')
    parts.append("</robot>")
    return "\n".join(parts)


class _T:
    """Builder of a parent list: chain(p, k) appends k links below p and returns the last one."""
    def __init__(self):
        self.parents = []

    def add(self, p):
        self.parents.append(p)
        return len(self.parents)

    def chain(self, p, k):
        for _ in range(k):
            p = self.add(p)
        return p


def _hand_made():
    """name -> (URDF text, floating).  Each reaches a branch of the partition / kernel that random trees may miss."""
    out = {}
    t = _T()                                       # six subtrees off a floating base: two roles own two subtrees each
    tips = [t.chain(0, 2) for _ in range(6)]
    out["six_subtrees"] = (_tree_urdf(t.parents, 1, geoms={**{x: "s" for x in tips}, 0: "s"}), True)
    t = _T()                                       # two branches: the trunk grows past the root, roles 2 and 3 own nothing
    a, b = t.chain(0, 3), t.chain(0, 3)
    out["two_branches"] = (_tree_urdf(t.parents, 2, geoms={a: "s", b: "c"}), True)
    t = _T()                                       # revolute, fixed and prismatic trunk joints before a 4-way branch
    t0 = t.add(0); t1 = t.add(t0); t2 = t.add(t1)
    tips = [t.chain(t2, 2) for _ in range(4)]
    out["fixed_prismatic_trunk"] = (_tree_urdf(t.parents, 3, joints={t1: "fixed", t2: "prismatic"},
                                               geoms={**{x: "s" for x in tips}, t1: "c"}), True)
    t = _T()                                       # a trunk link with a non-adjacent trunk child; geoms on base, trunk and subtrees
    t0 = t.add(0); t1 = t.add(t0)
    legs = [t.chain(t1, 2), t.chain(t1, 2)]
    t2 = t.add(t0)
    legs += [t.chain(t2, 2), t.chain(t2, 2)]
    out["nonadjacent_trunk_child"] = (_tree_urdf(t.parents, 4, geoms={0: "s", t0: "c", t2: "s", **{x: "s" for x in legs}}), True)
    t = _T()                                       # a subtree that branches: own-internal accumulator and xw slots
    r = t.add(0); u = t.chain(r, 2); v = t.chain(r, 2); w = t.chain(u - 1, 1)
    legs = [t.chain(0, 2) for _ in range(3)]
    out["branching_subtree"] = (_tree_urdf(t.parents, 5, geoms={u: "s", v: "c", w: "s", **{x: "s" for x in legs}}), True)
    t = _T()                                       # subtrees on a fixed base: their contribution to the base is dropped
    legs = [t.chain(0, 3) for _ in range(4)]
    out["fixed_base_subtrees"] = (_tree_urdf(t.parents, 6, geoms={x: "s" for x in legs}), False)
    t = _T()                                       # exactly TDS_TEAM_MAXK = 28 local links in role 0
    tip = t.chain(0, 28)
    legs = [t.add(0) for _ in range(3)]
    out["maxk_28"] = (_tree_urdf(t.parents, 7, geoms={tip: "s", tip - 14: "c", **{x: "s" for x in legs}}, reach=0.06), True)
    t = _T()                                       # TDS_TEAM_MAXC = 48 candidates: 24 capsules (TDS_MAX_GEOMS)
    legs = [t.chain(0, 3) for _ in range(4)]
    out["maxc_48"] = (_tree_urdf(t.parents, 8, geoms={i: "cc" for i in range(1, 13)}, reach=0.15), True)
    return out


def _maxk_29_urdf():
    t = _T()
    t.chain(0, 29)
    for _ in range(3):
        t.add(0)
    return _tree_urdf(t.parents, 9, reach=0.06)


# ---- models and states --------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _random_model(seed):
    rng = np.random.default_rng(31000 + seed)
    text = _random_urdf(rng, int(rng.integers(3, 24)), massless_links=False, boxes=False)
    return compile_urdf(text, PLANE if seed % 5 else None, floating=bool(seed % 2))


def _served(model):
    """True when the tree kernels serve the model: valid, and tds_build_team cuts it into a trunk and subtrees."""
    try:
        return emu_team.info(model)["rc"] == 0
    except RuntimeError:
        return False


@functools.lru_cache(maxsize=None)
def random_seeds():
    return tuple(s for s in RANDOM_SEEDS if _served(_random_model(s)))


HAND_MADE = tuple(_hand_made().keys())
FIXTURES = ("laikago", "ant", "humanoid")


def tree_ids():
    return [f"fixture-{f}" for f in FIXTURES] + [f"hand-{h}" for h in HAND_MADE] + [f"random-{s}" for s in random_seeds()]


@functools.lru_cache(maxsize=None)
def tree(tid, n=N):
    """(model, q, qd, tau) of tree `tid`: fp32-representable states; the base (a floating base) or the roots (a fixed base) lowered
    until geoms penetrate the plane in most environments, while every third environment of a floating base stays in the air."""
    kind, name = tid.split("-", 1)
    if kind == "fixture":
        model = np.array(load_model(fixture_path(name)))
    elif kind == "hand":
        text, floating = _hand_made()[name]
        model = compile_urdf(text, PLANE, floating=floating)
    else:
        model = _random_model(int(name)).copy()
    rng = np.random.default_rng(zlib.crc32(tid.encode()) if kind != "random" else 500 + int(name))
    n_links, floating, n_q, n_qd = int(model[1]), bool(model[2]), int(model[3]), int(model[4])
    q = np.zeros((n, n_q)); qd = rng.uniform(-1, 1, (n, n_qd)); tau = rng.uniform(-2, 2, (n, n_qd - (6 if floating else 0)))
    if floating:
        ax = rng.normal(size=(n, 3)); ax /= np.linalg.norm(ax, axis=1, keepdims=True)
        ang = rng.uniform(0, 0.6, n)
        q[:, :3], q[:, 3] = ax * np.sin(ang / 2)[:, None], np.cos(ang / 2)
        q[:, 4:6] = rng.uniform(-0.2, 0.2, (n, 2))
        qd[:, :6] *= 0.5
    for i in range(n_links):
        if int(_link(model, i, L_JTYPE)) != J_FIXED:
            q[:, int(_link(model, i, L_QIDX))] = rng.uniform(-0.8, 0.8, n)
    if model[7]:   # a plane: lower the tree into it
        P = port.make_params()
        f32 = lambda a: a.astype(np.float32).astype(np.float64)
        dmin = lambda m, i: min(port.step(m, P, 2, f32(q[i]), f32(qd[i]), None)["contact_data"][:, 9], default=np.inf)
        if floating:
            for i in range(n):
                d = dmin(model, i)
                if np.isfinite(d):
                    q[i, 6] = -d + (0.3 if i % 3 == 2 else -rng.uniform(0.003, 0.03))
        else:
            d = np.array([dmin(model, i) for i in range(n)])
            if np.isfinite(d).all():
                shift = np.median(d) + 0.01
                for i in range(n_links):
                    if int(_link(model, i, L_PARENT)) < 0:
                        model[H + BASE + i * LINK + L_XT_T + 2] -= shift
    q, qd, tau = (a.astype(np.float32).astype(np.float64) for a in (q, qd, tau))
    return model, q, qd, tau


@functools.lru_cache(maxsize=None)
def oracle(tid, mode):
    model, q, qd, tau = tree(tid)
    P = port.make_params()
    return [port.step(model, P, mode, q[i], qd[i], tau[i]) for i in range(q.shape[0])]


def out_key(mode):
    return ("qdd",) if mode == port.MODE_FD else ("q", "qd")


# ---- 1. fp64 against the C oracle, and the two maps against each other ---------------------------------------------------------
@pytest.mark.parametrize("tid", tree_ids())
def test_fp64_against_the_oracle(tid):
    """Both maps, both SMEM instances, the three modes: |x - ref| <= 2e-7 max(1, |ref|), or no worse than the world-frame kernel
    where that misses 2e-7 (the state is carried in fp32 between the stages of a step, in every kernel); in the full step also the signed distance
    of every candidate (the same penetrating set, distances within 1e-6) and the world transform of every link.  RoleWarps and
    LaneTeam sum over the roles in different orders: they must agree within 2e-7 relative on every output."""
    model, q, qd, tau = tree(tid)
    n_links = int(model[1])
    for mode in MODES:
        refs = oracle(tid, mode)
        world = emu.step(model, mode, q, qd, tau, precision=1)
        outs = {}
        for mp in ("role", "team"):
            for smem in (True, False):
                o = emu_team.step(model, mode, q, qd, tau, map=mp, precision=1, smem=smem)
                outs[mp, smem] = o
                for k in out_key(mode):
                    ref = np.array([r[k] for r in refs])
                    # (the humanoid's contact step: the world-frame kernel misses 2e-7 as well, 2.9e-7, through the fp32 state)
                    assert rel_err(o[k], ref) <= max(TOL64, rel_err(world[k], ref)), (mp, smem, mode, k)
                if mode == port.MODE_FULL and model[7]:
                    d_ref = np.array([r["contact_data"][:, 9] for r in refs])
                    assert o["contact_dist"].shape == d_ref.shape
                    assert np.array_equal(o["contact_dist"] < 0, d_ref < 0), (mp, smem)
                    assert np.max(np.abs(o["contact_dist"] - d_ref)) <= 1e-6, (mp, smem)
                    xf_ref = np.array([r["link_xf"] for r in refs]).reshape(-1, n_links, 12)
                    assert rel_err(o["link_xf"], xf_ref) <= 1e-6, (mp, smem)
        for k in out_key(mode) + ("contact_dist", "link_xf"):
            assert rel_err(outs["role", True][k], outs["team", True][k]) <= TOL64, (mode, k)


def test_every_served_tree_with_geoms_touches_and_rows_of_several_owners_interleave():
    """The states reach the contact solve: every tree with geoms on a plane has an environment with an active contact, and some
    environments have active rows of two or more owners (role warps then pass a barrier at every change of owner)."""
    multi = 0
    for tid in tree_ids():
        model, q, qd, tau = tree(tid)
        inf = emu_team.info(model)
        if not (model[7] and inf["n_cand"]):
            continue
        d = np.array([r["contact_data"][:, 9] for r in oracle(tid, port.MODE_FULL)])
        assert (d < 0).any(axis=1).any(), tid
        owners = [len(set(inf["cand_owner"][d[i] < 0])) for i in range(d.shape[0])]
        multi += sum(o >= 2 for o in owners)
    assert multi >= 10


# ---- 2. mixed and fp32 against their peer, the world-frame kernel ---------------------------------------------------------------
@pytest.mark.parametrize("tid", tree_ids())
def test_mixed_and_fp32_against_the_world_kernel(tid):
    """Mixed and fp32 arithmetic cannot meet 2e-7 and their error against the oracle depends on the tree's conditioning, so each
    is held to the host build of the world-frame kernel (tds_stepw.cu) in the same precision on the same states:
    err_tree <= C_MIXED * err_world + 1e-6.  Over every tree here, both maps and the three modes the worst observed ratio
    err_tree / err_world (where err_world > 1e-6) was 4.2 (random-19, forward dynamics, fp32 and mixed); C_MIXED = 6.
    One case is above 10: hand-nonadjacent_trunk_child, mixed, contact-free step, err_tree 1.7e-5 against err_world 8.3e-7
    (ratio 20).  Both kernels run the articulated-body pass in fp32 there; on the same states in forward dynamics the tree
    kernel's error (6.7e-5) is below the world kernel's (1.6e-4), so the ratio measures where each kernel's fp32 rounding lands
    on the largest velocities of these states, not a structural difference.  It is held to its own bound (MIXED_KNOWN)."""
    model, q, qd, tau = tree(tid)
    for precision in (0, 2):
        for mode in MODES:
            refs = oracle(tid, mode)
            w = emu.step(model, mode, q, qd, tau, precision=precision)
            for k in out_key(mode):
                ref = np.array([r[k] for r in refs])
                err_w = rel_err(w[k], ref)
                for mp in ("role", "team"):
                    o = emu_team.step(model, mode, q, qd, tau, map=mp, precision=precision)
                    err = rel_err(o[k], ref)
                    bound = MIXED_KNOWN.get((tid, precision, mode), C_MIXED * err_w + 1e-6)
                    assert err <= bound, (precision, mode, mp, k, err, err_w)


# ---- 4. bitwise invariants -------------------------------------------------------------------------------------------------------
BITWISE = [f"fixture-{f}" for f in FIXTURES] + [f"hand-{h}" for h in HAND_MADE]


def _same(a, b, keys=("q", "qd", "contact_dist", "link_xf")):
    return all(np.array_equal(a[k], b[k]) for k in keys)


@pytest.mark.parametrize("tid", BITWISE + ["random-bitwise"])
@pytest.mark.parametrize("precision", [0, 1])
def test_bitwise_invariants(tid, precision):
    """Indexing and synchronisation mistakes that a tolerance hides: the outputs of an environment are bit-identical whatever the
    batch around it (n = 1, 7, 9, 33, 37: ragged tiles of both maps; a permuted batch; tile neighbours in the air or on the
    ground), for the role-warp lane-by-lane mode with the tile-wide contact flag forced on or off and the exact 128-thread mode,
    for the shared-memory and the global-scratch instance, and for both orders in which the threads of a tile take turns."""
    if tid == "random-bitwise":
        tid = f"random-{random_seeds()[0]}"
    model, q, qd, tau = tree(tid)
    mode = port.MODE_FULL
    kw = dict(precision=precision)
    for mp in ("role", "team"):
        base = emu_team.step(model, mode, q, qd, tau, map=mp, **kw)
        sub = lambda o, idx: {k: o[k][idx] for k in ("q", "qd", "contact_dist", "link_xf")}
        for n in (1, 7, 9, 33, 37):
            assert _same(emu_team.step(model, mode, q[:n], qd[:n], tau[:n], map=mp, **kw), sub(base, slice(0, n))), (mp, n)
        perm = np.random.default_rng(3).permutation(q.shape[0])
        assert _same(emu_team.step(model, mode, q[perm], qd[perm], tau[perm], map=mp, **kw), sub(base, perm)), mp
        if model[7] and model[2]:   # environment 0 among neighbours lifted clear of the plane, then among neighbours that all touch
            air, ground = q.copy(), q.copy()
            air[1:, 6] += 5.0
            ground[2::3, 6] -= 0.31   # (tree(): every third environment is 0.3 above its first touch)
            for others, q2 in (("air", air), ("ground", ground)):
                o = emu_team.step(model, mode, q2, qd, tau, map=mp, **kw)
                assert _same(sub(o, slice(0, 1)), sub(base, slice(0, 1))), (mp, others)
        assert _same(emu_team.step(model, mode, q, qd, tau, map=mp, smem=False, **kw), base), (mp, "smem")
        assert _same(emu_team.step(model, mode, q, qd, tau, map=mp, descending=True, **kw), base), (mp, "descending")
    exact = emu_team.step(model, mode, q, qd, tau, map="role", **kw)
    for force_or in (False, True):
        lane = emu_team.step(model, mode, q, qd, tau, map="role", lane_by_lane=True, force_or=force_or, **kw)
        assert _same(lane, exact), force_or


# ---- 5. PD, reward, done and auto-reset -------------------------------------------------------------------------------------------
LOCO = {
    "laikago": dict(poses=envs.LAIKAGO_INITIAL_POSES, kp=envs.LAIKAGO_KP, kd=envs.LAIKAGO_KD, max_force=envs.LAIKAGO_MAX_FORCE),
    "ant": dict(poses=envs.ANT_INITIAL_POSES, kp=envs.ANT_KP, kd=envs.ANT_KD, max_force=envs.ANT_MAX_FORCE),
}


def _reward_done(kind, floating, q, qd):
    """The kernel's reward / done (tds_team_step.cuh) on the state after the step, and the margin of the done test."""
    q32, qd32 = q.astype(np.float32), qd.astype(np.float32)
    if kind == 2:
        up = np.ones(q.shape[0])
        if floating:
            qx, qy, qz, qw = (q[:, k] for k in range(4))
            up = 1 - 2 * (qx * qx + qy * qy) / (qx * qx + qy * qy + qz * qz + qw * qw)
        done = (up.astype(np.float32) < np.float32(0.6)) | (q32[:, 6] < np.float32(0.2))
        margin = np.minimum(np.abs(up - 0.6), np.abs(q[:, 6] - 0.2))
        return np.where(done, 0.0, q32[:, 4]), done, margin
    done = q32[:, 2] < np.float32(0.26)
    return np.where(done, 0.0, qd32[:, 0]), done, np.abs(q[:, 2] - 0.26)


@pytest.mark.parametrize("name", ["laikago", "ant"])
@pytest.mark.parametrize("reward_kind", [2, 3])
@pytest.mark.parametrize("mp", ["role", "team"])
def test_pd_env_step_on_the_fixtures_vs_locomotion_oracle(name, reward_kind, mp):
    """PD controller + full step against LocomotionContactSimulation restated by the oracle (as test_laikago_every_kernel_vs_c_oracle
    does on the GPU), reward and done of the kind asked for, and the auto-reset of the environments that report done."""
    model, q, qd, _ = tree(f"fixture-{name}")
    e = LOCO[name]
    n, n_q, n_act = q.shape[0], q.shape[1], len(e["poses"])
    act = np.random.default_rng(17).uniform(-0.6, 0.6, (n, n_act)).astype(np.float32).astype(np.float64)
    reset_q = np.linspace(-0.1, 0.1, n_q)
    env = emu_team.env_vector(model, n_act, 6, e["kp"], e["kd"], e["max_force"], 0.4, e["poses"], reward_kind, True, reset_q)
    o = emu_team.step(model, port.MODE_FULL, q, qd, act, map=mp, precision=1, use_pd=True, env=env)
    x = np.concatenate([q, qd, act, np.tile([e["kp"], e["kd"], e["max_force"]], (n, 1))], axis=1)
    ref = port.locomotion_step(model, port.make_params(), e["poses"], 6, x, 2048)
    rq, rqd = ref[:, :n_q], ref[:, n_q:2 * n_q]
    reward, done, margin = _reward_done(reward_kind, bool(model[2]), rq, rqd)
    clear = np.abs(margin) > 1e-5
    assert np.array_equal(o["done"][clear] > 0, done[clear])
    live = clear & ~done
    # (the kernel's PD controller runs in fp32, the locomotion oracle's in fp64: the bar of test_laikago_every_kernel_vs_c_oracle)
    assert rel_err(o["q"][live], rq[live]) <= 1e-5 and rel_err(o["qd"][live], rqd[live]) <= 1e-5
    assert np.max(np.abs(o["reward"][live] - reward[live]), initial=0) <= 1e-6 * max(1.0, np.max(np.abs(reward)))
    d = clear & done
    assert np.array_equal(o["q"][d], np.tile(reset_q.astype(np.float32), (d.sum(), 1))) and np.all(o["qd"][d] == 0)


def pd_setup(model, n, seed):
    """An actuator map over the non-fixed joints (tds_b200_set_env's rule), random poses and actions that the action limit clips."""
    rng = np.random.default_rng(seed)
    links = [i for i in range(int(model[1])) if int(_link(model, i, L_JTYPE)) != J_FIXED][:32]
    poses = rng.uniform(-0.3, 0.3, len(links))
    act = rng.uniform(-0.7, 0.7, (n, len(links))).astype(np.float32).astype(np.float64)
    return links, poses, act, dict(kp=30.0, kd=0.8, max_force=15.0, action_limit=0.5)


def pd_torques(model, links, poses, act, q, qd, kp, kd, max_force, action_limit):
    """tds_team_step.cuh's PD controller in fp32 (clip the action, kp, kd, max_force): the joint torques (no base dofs)."""
    f = np.float32
    off = 6 if model[2] else 0
    tau = np.zeros((q.shape[0], int(model[4]) - off))
    for k, li in enumerate(links):
        a = np.clip(act[:, k].astype(f), -f(action_limit), f(action_limit))
        q_des = f(poses[k]) + a
        qi, qdi = int(_link(model, li, L_QIDX)), int(_link(model, li, L_QDIDX))
        t = f(kp) * (q_des - q[:, qi].astype(f)) + f(kd) * (f(0) - qd[:, qdi].astype(f))
        tau[:, qdi - off] = np.clip(t, -f(max_force), f(max_force))
    return tau


@pytest.mark.parametrize("tid", [f"hand-{h}" for h in HAND_MADE] + ["random-pd"])
def test_pd_reward_done_and_auto_reset_on_trees(tid):
    """use_pd on trees with an actuator map over the non-fixed joints, reward kind 3 and auto-reset: the reference is the oracle
    driven with the PD torques computed in numpy."""
    seeds = random_seeds()
    for t in ([tid] if tid != "random-pd" else [f"random-{s}" for s in seeds[:8]]):
        model, q, qd, _ = tree(t)
        n, n_q = q.shape
        links, poses, act, g = pd_setup(model, n, 23)
        reset_q = np.linspace(0.05, 0.15, n_q)
        env = emu_team.env_vector(model, len(links), 0, g["kp"], g["kd"], g["max_force"], g["action_limit"], poses, 3, True, reset_q)
        P = port.make_params()
        tau = pd_torques(model, links, poses, act, q, qd, **g)
        refs = [port.step(model, P, port.MODE_FULL, q[i], qd[i], tau[i]) for i in range(n)]
        rq, rqd = np.array([r["q"] for r in refs]), np.array([r["qd"] for r in refs])
        reward, done, margin = _reward_done(3, bool(model[2]), rq, rqd)
        clear = np.abs(margin) > 1e-5
        for mp in ("role", "team"):
            o = emu_team.step(model, port.MODE_FULL, q, qd, act, map=mp, precision=1, use_pd=True, env=env)
            assert np.array_equal(o["done"][clear] > 0, done[clear]), (t, mp)
            live = clear & ~done
            assert rel_err(o["q"][live], rq[live]) <= TOL64 and rel_err(o["qd"][live], rqd[live]) <= TOL64, (t, mp)
            assert np.max(np.abs(o["reward"][live] - reward[live]), initial=0) <= 1e-6 * max(1.0, np.max(np.abs(reward))), (t, mp)
            d = clear & done
            assert np.array_equal(o["q"][d], np.tile(reset_q.astype(np.float32), (d.sum(), 1))) and np.all(o["qd"][d] == 0), (t, mp)


# ---- 6. capacity edges and coverage -----------------------------------------------------------------------------------------------
def test_29_local_links_in_one_role_are_refused():
    """One more local link than TDS_TEAM_MAXK: tds_build_team refuses the model (the library then runs the world-frame kernel)."""
    model = compile_urdf(_maxk_29_urdf(), PLANE, floating=True)
    assert emu_team.info(model)["rc"] == -1
    q = np.zeros((2, int(model[3]))); q[:, 3] = 1.0
    with pytest.raises(RuntimeError, match="rc=-3"):
        emu_team.step(model, 2, q, np.zeros((2, int(model[4]))))


def test_the_seeds_and_hand_made_trees_reach_every_structure():
    """Without this the random test could pass without reaching the cases it exists for."""
    infos = {tid: emu_team.info(tree(tid)[0]) for tid in tree_ids()}
    assert len(random_seeds()) >= 28
    reached = {
        "n_trunk >= 2": any(i["n_trunk"] >= 2 for i in infos.values()),
        "a role with several subtrees": any((i["subtrees"] > 1).any() for i in infos.values()),
        "a role with no own links": any((i["n_loc"] == i["n_trunk"]).any() for i in infos.values()),
        "n_xw_team > 0": any(i["n_xw_team"] > 0 for i in infos.values()),
        "n_xw_lane > 0": any(i["n_xw_lane"] > 0 for i in infos.values()),
        "an own-internal accumulator": any(i["own_internal"] > 0 for i in infos.values()),
        "a trunk-internal accumulator": any(i["trunk_internal"] > 0 for i in infos.values()),
        "candidates of every role": any(len(set(i["cand_owner"])) == 4 for i in infos.values()),
        "a fixed base with subtrees": any(not i["floating"] and i["dropped_subtrees"] > 0 for i in infos.values()),
        "kmax = 28": any(i["kmax"] == 28 for i in infos.values()),
        "n_cand = 48": any(i["n_cand"] == 48 for i in infos.values()),
        "a role-warp tile beyond shared memory": any(i["role_tile_bytes"][1] > 227 * 1024 for i in infos.values()),
    }
    print("reached: " + "; ".join(k for k, v in reached.items() if v))
    missing = [k for k, v in reached.items() if not v]
    assert not missing, missing
