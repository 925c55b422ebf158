"""Batched worlds of rigid bodies on the GPU: the RigidBody path of the reference's World::step (src/world.hpp:293-363,
src/rigid_body.hpp, src/rb_constraint_solver.hpp; python/examples/billiard_optimization.py steps exactly this loop).
Host side of csrc/tds_rigid.cu / the tds_b200_rigid_* C-ABI (include/tds_b200.h)."""
import ctypes

import numpy as np

from . import _lib

SPHERE, PLANE, CAPSULE, BOX = 0, 1, 2, 4     # tds::GeometryTypes (src/geometry.hpp:30-38)


def sphere(mass, radius):
    return [mass, SPHERE, radius, 0.0, 0.0, 0.0]


def capsule(mass, radius, length):
    return [mass, CAPSULE, radius, length, 0.0, 0.0]


def box(mass, extents):
    return [mass, BOX, extents[0], extents[1], extents[2], 0.0]


def plane(normal=(0.0, 0.0, 1.0), constant=0.0):
    return [0.0, PLANE, normal[0], normal[1], normal[2], constant]


# ---- per-world physical parameters (DESIGN.md section 7.11; ids in include/tds_b200.h) ----
_SIZE_NAMES = {SPHERE: ("radius",), CAPSULE: ("radius", "length"), BOX: ("extent_x", "extent_y", "extent_z")}


def _param_table(bodies):
    """[(id, name, model value)] of the parameter ids a world of these bodies has (friction and restitution: value None)."""
    d = np.asarray(bodies, dtype=np.float64).reshape(-1, 6)
    out = [(0, "friction", None), (1, "restitution", None)]
    for b, rec in enumerate(d):
        t = int(rec[1])
        if t == PLANE:
            continue
        if rec[0] != 0.0:
            out.append((2 + 4 * b, f"body{b}.mass", float(rec[0])))
        for c, nm in enumerate(_SIZE_NAMES[t]):
            out.append((2 + 4 * b + 1 + c, f"body{b}.{nm}", float(rec[2 + c])))
    return out


def param_names(bodies):
    """Names of the physical parameters a world of these bodies has, in id order: "friction", "restitution", "body<b>.mass" (dynamic
    bodies), "body<b>.radius" (spheres, capsules), "body<b>.length" (capsules), "body<b>.extent_x" / _y / _z (boxes).  Host only."""
    return [nm for _, nm, _ in _param_table(bodies)]


def param_values(bodies, friction=0.5, restitution=0.0):
    """The description's value of every parameter of param_names(bodies) (float64, same order); friction and restitution are the
    world settings given (RigidWorld's defaults unless stated).  Host only."""
    return np.asarray([(friction if i == 0 else restitution) if v is None else v for i, _, v in _param_table(bodies)], dtype=np.float64)


def param_ids(bodies, names_or_ids):
    """Parameter names (param_names) and / or ids -> list of int ids (ValueError for an unknown name; ids are checked on install)."""
    table = {nm: i for i, nm, _ in _param_table(bodies)}
    ids = []
    for x in names_or_ids:
        if isinstance(x, str):
            if x not in table:
                raise ValueError(f"unknown physical parameter {x!r}")
            ids.append(table[x])
        else:
            ids.append(int(x))
    return ids


def identity_state(n_worlds, n_bodies):
    """[n_worlds][n_bodies][13]: everything zero, orientations the identity quaternion (x, y, z, w) = (0, 0, 0, 1)."""
    s = np.zeros((n_worlds, n_bodies, 13))
    s[:, :, 6] = 1.0
    return s


class RigidWorld:
    """n_worlds independent worlds of the same bodies.  bodies: list of sphere() / capsule() / box() / plane() records, in the
    order the reference's World would hold them (contacts are enumerated over pairs i < j in that order)."""

    def __init__(self, bodies, n_worlds, device=0, **params):
        self._L = _lib.lib()
        self.desc = np.ascontiguousarray(bodies, dtype=np.float64).reshape(-1, 6)
        self.n_bodies, self.n_worlds, self.device = self.desc.shape[0], int(n_worlds), device
        self._h = self._L.tds_b200_rigid_create(ctypes.c_void_p(self.desc.ctypes.data), self.n_bodies, self.n_worlds, device)
        if not self._h:
            raise RuntimeError("tds_b200_rigid_create: " + _lib.last_error())
        self.param_ids = []   # installed physical parameters (set_physical_params)
        self.set_params(**params)

    def close(self):
        if getattr(self, "_h", None):
            self._L.tds_b200_rigid_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc, what):
        if rc:
            raise RuntimeError(f"{what}: rc={rc} {_lib.last_error()}")

    def set_params(self, dt=1.0 / 60.0, gravity=(0.0, 0.0, -9.81), friction=0.5, restitution=0.0, erp=0.1, num_solver_iterations=1):
        g = np.asarray(gravity, dtype=np.float64)
        self._check(self._L.tds_b200_rigid_set_params(self._h, dt, ctypes.c_void_p(g.ctypes.data), friction, restitution, erp,
                                                      int(num_solver_iterations)), "rigid_set_params")

    def _args(self, state, force):
        s = np.ascontiguousarray(state, dtype=np.float64)
        assert s.shape == (self.n_worlds, self.n_bodies, 13), s.shape
        f = None
        if force is not None:
            f = np.ascontiguousarray(force, dtype=np.float64)
            assert f.shape == (self.n_worlds, self.n_bodies, 3), f.shape
        return s, f

    def step(self, state, force=None, steps=1):
        """`steps` calls of World::step(dt); force = apply_central_force before the first one.  Returns the new state."""
        s, f = self._args(state, force)
        out = np.zeros_like(s)
        self._check(self._L.tds_b200_rigid_step_host(self._h, ctypes.c_void_p(s.ctypes.data), ctypes.c_void_p(f.ctypes.data) if f is not None else None,
                                                     int(steps), ctypes.c_void_p(out.ctypes.data)), "rigid_step_host")
        return out

    def step_jacobian(self, state, force=None, steps=1):
        """(state_out, J): J [n_worlds][13 n_bodies][16 n_bodies] = d state_out / d (state | force), forward-mode on the GPU."""
        s, f = self._args(state, force)
        out = np.zeros_like(s)
        jac = np.zeros((self.n_worlds, 13 * self.n_bodies, 16 * self.n_bodies))
        self._check(self._L.tds_b200_rigid_jacobian_host(self._h, ctypes.c_void_p(s.ctypes.data), ctypes.c_void_p(f.ctypes.data) if f is not None else None,
                                                         int(steps), ctypes.c_void_p(out.ctypes.data), ctypes.c_void_p(jac.ctypes.data)), "rigid_jacobian_host")
        return out, jac

    def step_vjp(self, state, force, g_state_out, steps=1):
        """(g_state, g_force) = g_state_out^T d state_out / d (state, force) of `steps` World::step calls, by reverse mode on the
        GPU (one recorded step at a time, the states checkpointed on the device).  Host arrays [n_worlds][n_bodies][13 | 3]."""
        s, f = self._args(state, force)
        g = np.ascontiguousarray(g_state_out, dtype=np.float64)
        assert g.shape == s.shape, g.shape
        gs, gf = np.zeros_like(s), np.zeros((self.n_worlds, self.n_bodies, 3))
        v = lambda a: ctypes.c_void_p(a.ctypes.data) if a is not None else None
        self._check(self._L.tds_b200_rigid_vjp_host(self._h, v(s), v(f), int(steps), v(g), v(gs), v(gf)), "rigid_vjp_host")
        return gs, gf

    def step_vjp_device(self, state, force, g_state_out, g_state, g_force=None, steps=1, stream=None):
        """Device version of step_vjp: float64 CUDA tensors state / g_state_out / g_state [13 * n_bodies][n_stride], force / g_force
        [3 * n_bodies][n_stride] (force None: zero force; g_force None: not computed).  stream None = the world's own stream.
        Synchronous."""
        p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
        self._check(self._L.tds_b200_rigid_vjp_device(self._h, p(state), p(force), int(steps), p(g_state_out), p(g_state), p(g_force),
                                                      ctypes.c_void_p(stream.cuda_stream) if stream is not None else None), "rigid_vjp_device")

    def step_jvp(self, state, force=None, t_state=None, t_force=None, steps=1, t_par=None):
        """(state_out, t_state_out): Jacobian-vector products of `steps` World::step calls by forward mode on the GPU, one launch for
        the whole rollout.  t_state [n_worlds][n_bodies][13][m], t_force [n_worlds][n_bodies][3][m], t_par [n_worlds][k][m] (tangents
        of the installed parameters; any may be None; without the trailing m axis: m = 1, and t_state_out then comes back without it
        too).  t_state_out [n_worlds][n_bodies][13][m]."""
        s, f = self._args(state, force)
        first = next((x for x in (t_state, t_force) if x is not None), None)
        single = np.ndim(first) == 3 if first is not None else (t_par is not None and np.ndim(t_par) == 2)

        def prep(x, shape):
            if x is None:
                return None
            x = np.asarray(x, dtype=np.float64)
            if x.ndim == len(shape):
                x = x[..., None]
            assert x.shape[:len(shape)] == shape, x.shape
            return np.ascontiguousarray(x)
        ts, tf = prep(t_state, (self.n_worlds, self.n_bodies, 13)), prep(t_force, (self.n_worlds, self.n_bodies, 3))
        tp = prep(t_par, (self.n_worlds, len(self.param_ids)))
        m = next((x.shape[-1] for x in (ts, tf, tp) if x is not None), 0)
        out = np.zeros_like(s)
        t_out = np.zeros((self.n_worlds, self.n_bodies, 13, max(m, 1)))
        v = lambda a: ctypes.c_void_p(a.ctypes.data) if a is not None else None
        if tp is None:
            self._check(self._L.tds_b200_rigid_jvp_host(self._h, v(s), v(f), int(steps), m, v(ts), v(tf), v(out), v(t_out)), "rigid_jvp_host")
        else:
            self._check(self._L.tds_b200_rigid_jvp_params_host(self._h, v(s), v(f), int(steps), m, v(ts), v(tf), v(tp), v(out), v(t_out)),
                        "rigid_jvp_params_host")
        return out, (t_out[..., 0] if single else t_out)

    def step_jvp_device(self, state, force, m, t_state, t_force, state_out, t_state_out, steps=1, stream=None, t_par=None):
        """Device version of step_jvp: float64 CUDA tensors state [13 * n_bodies][n_stride], force [3 * n_bodies][n_stride] or None,
        t_state / t_state_out [13 * n_bodies * m][n_stride], t_force [3 * n_bodies * m][n_stride], t_par [k * m][n_stride] (entry (r, j)
        at row r * m + j; any tangent may be None), state_out [13 * n_bodies][n_stride] or None (not state itself).  stream None = the
        world's own stream.  Asynchronous."""
        p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
        st = ctypes.c_void_p(stream.cuda_stream) if stream is not None else None
        if t_par is None:
            self._check(self._L.tds_b200_rigid_jvp_device(self._h, p(state), p(force), int(steps), int(m), p(t_state), p(t_force), p(state_out),
                                                          p(t_state_out), st), "rigid_jvp_device")
        else:
            self._check(self._L.tds_b200_rigid_jvp_params_device(self._h, p(state), p(force), int(steps), int(m), p(t_state), p(t_force),
                                                                 p(t_par), p(state_out), p(t_state_out), st), "rigid_jvp_params_device")

    # ---- per-world physical parameters (DESIGN.md section 7.11) ----
    def set_physical_params(self, names_or_ids, values=None, stream=None):
        """Install physical parameters per world: names (param_names) or ids, and values float64 [n_worlds, k] or [k] (every world), a
        numpy array (checked, synchronous) or a CUDA tensor (copied on `stream`, default torch's current stream, without checks).
        names_or_ids None (or empty) clears the set.  Every step, Jacobian, VJP and JVP then uses each world's values for these
        parameters and the description's for the rest."""
        ids = [] if names_or_ids is None else param_ids(self.desc, names_or_ids)
        k = len(ids)
        idv = np.ascontiguousarray(ids, dtype=np.int32)
        idp = ctypes.c_void_p(idv.ctypes.data) if k else None
        if k == 0:
            self._check(self._L.tds_b200_rigid_set_physical_params_host(self._h, 0, None, None), "rigid_set_physical_params")
        elif hasattr(values, "is_cuda") and values.is_cuda:
            import torch
            v = values.detach().to(torch.float64)
            if v.dim() == 1:
                v = v.unsqueeze(0).expand(self.n_worlds, k)
            if tuple(v.shape) != (self.n_worlds, k):
                raise ValueError(f"values: [n_worlds, {k}] or [{k}] expected, got {tuple(values.shape)}")
            soa = torch.zeros((k, self.n_stride), dtype=torch.float64, device=v.device)
            soa[:, :self.n_worlds] = v.t()
            # (the C-ABI reads torch's default stream, handle NULL, as the world's own stream: copy on a side stream ordered after
            # torch's current one; without a stream given, wait for the copy, since later calls may run on any stream)
            st = stream if stream is not None else torch.cuda.Stream(v.device)
            st.wait_stream(torch.cuda.current_stream(v.device))
            self._check(self._L.tds_b200_rigid_set_physical_params_device(self._h, k, idp, ctypes.c_void_p(soa.data_ptr()),
                                                                          ctypes.c_void_p(st.cuda_stream)), "rigid_set_physical_params")
            if stream is None:
                st.synchronize()
            else:
                soa.record_stream(st)
        else:
            v = np.asarray(values, dtype=np.float64)
            if v.ndim == 1:
                v = np.broadcast_to(v, (self.n_worlds, k))
            if v.shape != (self.n_worlds, k):
                raise ValueError(f"values: [n_worlds, {k}] or [{k}] expected, got {v.shape}")
            v = np.ascontiguousarray(v)
            self._check(self._L.tds_b200_rigid_set_physical_params_host(self._h, k, idp, ctypes.c_void_p(v.ctypes.data)),
                        "rigid_set_physical_params")
        self.param_ids = ids

    def param_count(self):
        """Number of parameter ids of the world, 2 + 4 n_bodies (not all of them exist: see param_names)."""
        return self._L.tds_b200_rigid_param_count(self._h)

    def step_param_jacobian(self, state, force=None, steps=1):
        """(state_out, J_par): J_par [n_worlds][13 n_bodies][k] = d state_out / d (installed parameters) of `steps` World::step calls,
        forward-mode on the GPU, columns in the order of set_physical_params."""
        s, f = self._args(state, force)
        out = np.zeros_like(s)
        jac = np.zeros((self.n_worlds, 13 * self.n_bodies, len(self.param_ids)))
        v = lambda a: ctypes.c_void_p(a.ctypes.data) if a is not None else None
        self._check(self._L.tds_b200_rigid_param_jacobian_host(self._h, v(s), v(f), int(steps), v(out), v(jac)), "rigid_param_jacobian_host")
        return out, jac

    def step_vjp_params(self, state, force, g_state_out, steps=1):
        """step_vjp with the installed parameters as further inputs: (g_state, g_force, g_par [n_worlds][k]); g_par is summed over
        the `steps` steps."""
        s, f = self._args(state, force)
        g = np.ascontiguousarray(g_state_out, dtype=np.float64)
        assert g.shape == s.shape, g.shape
        gs, gf = np.zeros_like(s), np.zeros((self.n_worlds, self.n_bodies, 3))
        gp = np.zeros((self.n_worlds, len(self.param_ids)))
        v = lambda a: ctypes.c_void_p(a.ctypes.data) if a is not None else None
        self._check(self._L.tds_b200_rigid_vjp_params_host(self._h, v(s), v(f), int(steps), v(g), v(gs), v(gf), v(gp)), "rigid_vjp_params_host")
        return gs, gf, gp

    def step_vjp_params_device(self, state, force, g_state_out, g_state, g_force, g_par, steps=1, stream=None):
        """Device version of step_vjp_params: as step_vjp_device, and g_par [k][n_stride] float64 CUDA tensor.  Synchronous."""
        p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
        self._check(self._L.tds_b200_rigid_vjp_params_device(self._h, p(state), p(force), int(steps), p(g_state_out), p(g_state), p(g_force),
                                                             p(g_par), ctypes.c_void_p(stream.cuda_stream) if stream is not None else None),
                    "rigid_vjp_params_device")

    def step_device(self, state_in, state_out, force=None, steps=1, stream=None):
        """CUDA tensors, fp64: state [13 * n_bodies][n_stride], force [3 * n_bodies][n_stride] or None; in place allowed."""
        p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
        self._check(self._L.tds_b200_rigid_step_device(self._h, p(state_in), p(state_out), p(force), int(steps),
                                                       ctypes.c_void_p(stream.cuda_stream) if stream is not None else None), "rigid_step_device")

    @property
    def n_stride(self):
        return (self.n_worlds + 31) & ~31
