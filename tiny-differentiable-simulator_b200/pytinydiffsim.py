"""The `pytinydiffsim` names of the hot path, served by libtds_b200.so (python/pytinydiffsim.inl of the reference):

    TinyWorld (.step, .gravity, .friction, .restitution)                      pytinydiffsim.inl:857-876
    TinyMultiBody (.q .qd .qdd .tau, is_floating, num_dofs, clear_forces)     :611-655
    TinyUrdfParser.load_urdf, UrdfToMultiBody2.convert2                       :1013-1034
    forward_dynamics(mb, gravity), integrate_euler(mb, dt), integrate_euler_qdd(mb, dt)   :659-663
    mass_matrix(mb[, q])                                                      :659-663 (mass_matrix.hpp)
    point_jacobian(mb, link_index, point, is_local_point=False)               (jacobian.hpp:85-90)
    inverse_dynamics(mb, q, qd, qdd, gravity), bias_forces(mb, q, qd, gravity)   (inverse_dynamics.hpp)
    VectorizedLaikagoEnv, VectorizedAntEnv (pytinydiffsim_includes.h:58-227), CartpoleEnv (:1123)

The fine-grained calls operate on one MultiBody like the reference's; each is one stage of the GPU path (forward dynamics =
MODE_FD of the step kernel, World.step = MODE_WORLD, the two integrators = the integration kernels), so a script written as

    pd.forward_dynamics(mb, world.gravity); pd.integrate_euler_qdd(mb, dt); world.step(dt); pd.integrate_euler(mb, dt)

runs unchanged - at per-call host<->device cost.  The fast path for many environments is tds_b200.BatchSim /
VectorizedLaikagoEnv, which fuse the same sequence into one kernel.  There is no CPU fallback: without the library or a GPU
every compute call raises.
"""
import numpy as np

from . import _lib
from . import rigid as _rigid
from .envs import VectorizedLaikagoEnv, VectorizedLaikagoEnvOutput, VectorizedAntEnv  # noqa: F401
from .model import compile_urdf, fixture_path, load_model, merge_models
from .sim import BatchSim, MODE_FD, MODE_NOCONTACT, MODE_FULL, MODE_WORLD


class TinyUrdfStructures:
    def __init__(self, source=""):
        self.source = source            # file path or URDF text
        self.robot_name = ""
        self.is_plane = "<plane" in (source if source.lstrip().startswith("<") else open(source).read()) if source else False


class TinyUrdfParser:
    def load_urdf(self, file_name):
        return TinyUrdfStructures(file_name)


class TinyWorld:
    def __init__(self):
        self.gravity = (0.0, 0.0, -9.81)
        self.friction = 0.5               # World::default_friction, src/world.hpp:68
        self.restitution = 0.0
        self.num_solver_iterations = 1    # World::num_solver_iterations, src/world.hpp:65 (sweeps of the rigid-body solver; the multibody LCP does not use it)
        self.pgs_iterations, self.erp, self.cfm, self.keep_all_points = 1, 0.2, 1e-5, False   # mb_constraint_solver.hpp:59-70
        self._plane = None                # URDF of the static plane body (created first, like the locomotion envs do)
        self._bodies = []

    def step(self, dt):
        """World::step (src/world.hpp:302-363): contact detection + constraint solve.  One multibody: against the plane.  Several
        fixed-base multibodies (one root link each): ONE simulator over the merged model (tds_b200.model.merge_models), so that
        the contacts between multibodies (sphere-sphere, capsule-sphere, :206-282) are found and solved list after list like the
        reference does.  A world mixing in floating-base multibodies steps each against the plane only."""
        bodies = self._bodies
        if len(bodies) > 1 and all(not b._floating and b._single_root() for b in bodies):
            key = tuple(id(b) for b in bodies)
            if getattr(self, "_merged_key", None) != key:
                self._merged = BatchSim(merge_models([b._model for b in bodies]), 1, precision=1)
                self._merged_key = key
            sim = self._merged
            sim.set_params(dt, self.gravity, self.friction, self.restitution, self.erp, self.cfm, self.pgs_iterations, self.keep_all_points)
            q = np.concatenate([b.q for b in bodies]); qd = np.concatenate([b.qd for b in bodies])
            out = sim.step_host(MODE_WORLD, q[None], qd[None], None)["qd"][0]
            o = 0
            for b in bodies:
                b.qd = out[o:o + b.qd.size].copy()
                o += b.qd.size
            return
        for mb in bodies:
            mb._world_step(self, dt)


class TinyMultiBody:
    def __init__(self, floating=False):
        self._floating = bool(floating)
        self._sim = None
        self.q = self.qd = self.qdd = self.tau = None
        self.links = []

    def is_floating(self):
        return self._floating

    def _single_root(self):
        m = self._model
        n_links = int(m[1])
        parents = m[16 + 13:16 + 13 + n_links * 34:34]
        return int(np.sum(parents < 0)) == 1

    @property
    def num_dofs(self):
        return self._sim.n_q

    def initialize(self):
        pass

    def clear_forces(self):
        """MultiBody::clear_forces (multi_body.hpp:578-586): zeroes tau (and the applied forces, which the path does not use)."""
        self.tau[:] = 0.0

    def set_q(self, q):
        self.q[:] = np.asarray(q, dtype=np.float64)

    # -- stages -------------------------------------------------------------------------------------------------
    def _bind(self, sim):
        self._sim = sim
        self.q = np.zeros(sim.n_q)
        if self._floating:
            self.q[3] = 1.0
        self.qd, self.qdd, self.tau = np.zeros(sim.n_qd), np.zeros(sim.n_qd), np.zeros(sim.n_tau)
        self.links = [None] * sim.n_links

    def _params(self, world=None, dt=None, gravity=None):
        s = self._sim
        w = world or self._world
        s.set_params(dt if dt is not None else s.dt, gravity if gravity is not None else w.gravity, w.friction, w.restitution,
                     w.erp, w.cfm, w.pgs_iterations, w.keep_all_points)

    def _forward_dynamics(self, gravity):
        self._params(gravity=tuple(np.asarray(gravity, dtype=np.float64)))
        out = self._sim.step_host(MODE_FD, self.q[None], self.qd[None], self.tau[None] if self.tau.size else None)
        self.qdd = out["qdd"][0].copy()

    def _world_step(self, world, dt):
        self._params(world=world, dt=dt)
        out = self._sim.step_host(MODE_WORLD, self.q[None], self.qd[None], None)
        self.qd = out["qd"][0].copy()

    def _integrate(self, dt, update_q):
        self._params(dt=dt)
        self.q, self.qd = self._sim.integrate_host(self.q, self.qd, self.qdd, update_q)
        if not update_q:
            self.qdd = np.zeros_like(self.qdd)      # integrate_euler_qdd zeroes qdd (integrator.hpp:194)


class UrdfToMultiBody2:
    def convert2(self, urdf_structures, world, mb):
        """UrdfToMultiBody::convert_to_multi_body (src/urdf/urdf_to_multi_body.hpp:41): here the model compiler
        (tds_b200_urdf_to_model) + a one-environment simulator on the GPU."""
        if urdf_structures.is_plane:
            world._plane = urdf_structures.source
            return True
        model = compile_urdf(urdf_structures.source, world._plane, mb.is_floating())
        mb._world = world
        mb._model = model
        mb._bind(BatchSim(model, 1, precision=1))    # strict fp64 arithmetic: a single body is not a throughput case
        world._bodies.append(mb)
        return True


def forward_dynamics(mb, gravity):
    mb._forward_dynamics(gravity)


def integrate_euler(mb, dt):
    mb._integrate(dt, True)


def integrate_euler_qdd(mb, dt):
    mb._integrate(dt, False)


def mass_matrix(mb, q=None):
    """The joint-space mass matrix M(q) of the multibody: a NumPy float64 [num_dofs, num_dofs] array (qd-dimension, both triangles),
    by the CRBA of the GPU step in fp64 at the fp32-rounded q.  The reference's C++ call mass_matrix(mb, &M) reads the multibody's
    own q (mass_matrix.hpp:36, forward kinematics with an empty qd); its binding is served here in both forms: mass_matrix(mb) at
    mb.q, and mass_matrix(mb, q) at a q given explicitly (mb.q is left as it is)."""
    qv = np.asarray(mb.q if q is None else q, dtype=np.float64).reshape(1, -1)
    return mb._sim.mass_matrix_host(qv)[0]


def inverse_dynamics(mb, q, qd, qdd, gravity):
    """The joint forces tau for which the multibody has the accelerations qdd at (q, qd) under `gravity`: a NumPy float64 [num_dofs]
    array, by the recursive Newton-Euler algorithm of the GPU path in fp64 at the fp32-rounded inputs (DESIGN.md section 7.14).  A
    floating base's 6 rows are the wrench on the base in the base frame for the base-frame acceleration qdd[0:6], gravity rotated into
    the base frame.  The reference's Python binding of it is not pinned here; this follows the C++ free function
    inverse_dynamics(mb, q, qd, qdd, gravity) of inverse_dynamics.hpp.  mb is left as it is."""
    mb._params(gravity=tuple(np.asarray(gravity, dtype=np.float64)))
    row = lambda x: np.asarray(x, dtype=np.float64).reshape(1, -1)
    return mb._sim.inverse_dynamics_host(row(q), row(qd), row(qdd))[0]


def bias_forces(mb, q, qd, gravity):
    """The bias forces h(q, qd) = inverse_dynamics(mb, q, qd, 0, gravity): a NumPy float64 [num_dofs] array.  Follows the C++ free
    function bias_forces(mb, q, qd, gravity) of inverse_dynamics.hpp.  mb is left as it is."""
    mb._params(gravity=tuple(np.asarray(gravity, dtype=np.float64)))
    row = lambda x: np.asarray(x, dtype=np.float64).reshape(1, -1)
    return mb._sim.inverse_dynamics_host(row(q), row(qd), None)[0]


def point_jacobian(mb, link_index, point, is_local_point=False):
    """The 3 x num_dofs linear Jacobian of a point on link `link_index` (-1: the base) at mb.q: a NumPy float64 array, the reference's
    point_jacobian2(mb, link_index, point, is_local_point) (jacobian.hpp:85-90), computed by the kinematics of the GPU step in fp64 at the
    fp32-rounded q.  The reference's Python binding of it is not pinned here; this follows the C++ signature.  `point` is in the link's
    frame when is_local_point, else in world coordinates; a world point is mapped into the link's frame with the link's transform from
    the same kernel.  A floating base gives the reference's columns [-[x - r0]x^T | I3] (its rotation ignored)."""
    qv = np.asarray(mb.q, dtype=np.float64).reshape(1, -1)
    sim = mb._sim
    link = int(link_index)
    if not -1 <= link < sim.n_links:
        raise IndexError(f"link_index {link} out of [-1, {sim.n_links})")
    pt = np.asarray(point, dtype=np.float64).reshape(3)
    if not is_local_point:
        if link >= 0:
            R, p, _, _ = sim.kinematics_host(qv, [], np.zeros((0, 3)))
            R, p = R[0, link], p[0, link]
        else:   # the base's transform: its origin and axes as points of the base
            _, _, x, _ = sim.kinematics_host(qv, [-1] * 4, np.vstack([np.zeros(3), np.eye(3)]))
            p = x[0, 0]
            R = (x[0, 1:] - p).T
        pt = R.T @ (pt - p)
    return sim.kinematics_host(qv, [link], pt.reshape(1, 3))[3][0, 0]


# ---- rigid bodies (python/pytinydiffsim.inl:336-385, 448-455; examples/billiard_optimization.py) --------------------------------
class TinySphere:
    def __init__(self, radius):
        self._record = lambda mass: _rigid.sphere(mass, float(radius))
        self._radius = float(radius)

    def get_radius(self):
        return self._radius


class TinyCapsule:
    def __init__(self, radius, length):
        self._record = lambda mass: _rigid.capsule(mass, float(radius), float(length))
        self._radius, self._length = float(radius), float(length)

    def get_radius(self):
        return self._radius

    def get_length(self):
        return self._length


class TinyPlane:
    def __init__(self):
        self._record = lambda mass: _rigid.plane()

    def get_normal(self):
        return (0.0, 0.0, 1.0)

    def get_constant(self):
        return 0.0


class TinyPose:
    def __init__(self, position=(0.0, 0.0, 0.0), orientation=(0.0, 0.0, 0.0, 1.0)):
        self.position, self.orientation = list(position), list(orientation)     # orientation: quaternion x, y, z, w


class TinyRigidBody:
    """RigidBody (src/rigid_body.hpp): state holder on the host; the arithmetic runs on the GPU in rigid_world_step."""

    def __init__(self, mass, geometry):
        self.mass, self.collision_geometry = float(mass), geometry
        self.world_pose = TinyPose()
        self.linear_velocity, self.angular_velocity = [0.0, 0.0, 0.0], [0.0, 0.0, 0.0]
        self.total_force = [0.0, 0.0, 0.0]

    def apply_central_force(self, force):
        self.total_force = [a + float(b) for a, b in zip(self.total_force, force)]

    def clear_forces(self):
        self.total_force = [0.0, 0.0, 0.0]


def rigid_world_step(world, bodies, dt, steps=1):
    """The stepping loop of python/examples/billiard_optimization.py:118-131 (= World::step on rigid bodies, src/world.hpp:293-363)
    as ONE call: apply_gravity / apply_force_impulse / clear_forces, compute_contacts_rigid_body, num_solver_iterations sweeps of
    resolve_collision over the contacts, integrate - `steps` times, on the GPU (csrc/tds_rigid.cu).  Updates the bodies in place."""
    key = tuple(id(b) for b in bodies)
    if getattr(world, "_rigid_key", None) != key:
        world._rigid = _rigid.RigidWorld([b.collision_geometry._record(b.mass) for b in bodies], 1)
        world._rigid_key = key
    world._rigid.set_params(dt=dt, gravity=tuple(world.gravity), friction=world.friction, restitution=world.restitution,
                            num_solver_iterations=world.num_solver_iterations)
    state = np.array([[list(b.world_pose.position) + list(b.world_pose.orientation) + list(b.linear_velocity) + list(b.angular_velocity)
                       for b in bodies]], dtype=np.float64)
    force = np.array([[b.total_force for b in bodies]], dtype=np.float64)
    out = world._rigid.step(state, force, steps)[0]
    for b, s in zip(bodies, out):
        b.world_pose.position, b.world_pose.orientation = list(s[0:3]), list(s[3:7])
        b.linear_velocity, b.angular_velocity = list(s[7:10]), list(s[10:13])
        b.clear_forces()


class CartpoleEnvOutput:
    def __init__(self):
        self.obs, self.reward, self.done = [], 0.0, False


class CartpoleEnv:
    """pytinydiffsim.CartpoleEnv (examples/environments/cartpole_environment2.h:160-330): cartpole.urdf, dt 1/60, g -10,
    pipeline forward_dynamics -> integrate_euler (no World::step), action clipped to +-10, reward 1, done when |x| > 0.4
    or |theta| > 12 degrees."""

    def __init__(self, device=0, seed=0):
        self.sim = BatchSim(load_model(fixture_path("cartpole")), 1, device=device, dt=1.0 / 60.0, gravity=(0.0, 0.0, -10.0), precision=1)
        self.rng = np.random.default_rng(seed)
        self.sim_state = np.zeros(4)
        self.action_low_, self.action_high_ = -10.0, 10.0

    def seed(self, s):
        self.rng = np.random.default_rng(int(s))

    def reset(self):
        self.sim_state = 0.05 * (self.rng.random(4) - 0.5) * 2.0
        return list(self.sim_state)

    def step(self, action):
        a = float(min(max(action, self.action_low_), self.action_high_))
        out = self.sim.step_host(MODE_NOCONTACT, self.sim_state[None, :2], self.sim_state[None, 2:], np.array([[a, 0.0]]))
        self.sim_state = np.concatenate([out["q"][0], out["qd"][0]])
        o = CartpoleEnvOutput()
        o.obs = list(self.sim_state)
        o.reward = 1.0
        x, theta = self.sim_state[0], self.sim_state[1]
        o.done = bool(x < -0.4 or x > 0.4 or abs(theta) > 12.0 * 2.0 * np.pi / 360.0)
        return o


def lib_path():
    return _lib.lib_path()
