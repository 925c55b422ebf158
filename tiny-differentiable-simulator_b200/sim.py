"""BatchSim: N independent copies of World{plane, MultiBody} resident on one GPU.

Python-side mirror of the fine-grained pytinydiffsim surface for the hot path
(forward_dynamics / integrate_euler_qdd / TinyWorld.step / integrate_euler,
python/pytinydiffsim.inl:659-663,857-876), batched: one call = one step of all environments.
torch is used for device memory and streams only.
"""
import ctypes

import numpy as np

from . import _lib
from .model import model_dims

MODE_FD, MODE_NOCONTACT, MODE_FULL = 0, 1, 2
MODE_WORLD = 3   # World::step(dt) alone (src/world.hpp:293-363): contacts + constraint solve on (q, qd) -> qd; world-frame kernel
PREC_MIXED, PREC_F64, PREC_F32, PREC_AUTO = 0, 1, 2, -1


def _dp(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_double)) if a is not None else None


def _ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _stream(stream):
    """The CUDA stream handle of a device call: `stream`, or torch's current stream when None."""
    import torch
    return ctypes.c_void_p(stream.cuda_stream if stream is not None else torch.cuda.current_stream().cuda_stream)


def _sym3(c):
    """[..., 3, 3] symmetric matrices from their components [..., 6] (xx, xy, xz, yy, yz, zz)."""
    return c[..., [0, 1, 2, 1, 3, 4, 2, 4, 5]].reshape(c.shape[:-1] + (3, 3))


class BatchSim:
    def __init__(self, model, n_envs, device=0, dt=1e-3, gravity=(0.0, 0.0, -9.81), friction=0.5,
                 restitution=0.0, erp=0.2, cfm=1e-5, pgs_iterations=1, keep_all_points=False,
                 precision=PREC_AUTO):
        self._L = _lib.lib()
        self.model = np.ascontiguousarray(model, dtype=np.float64)
        self.info = model_dims(self.model)
        self._h = self._L.tds_b200_create(_dp(self.model), self.model.size, int(n_envs), int(device))
        if not self._h:
            raise RuntimeError("tds_b200_create failed: " + _lib.last_error())
        dims = (ctypes.c_int * 8)()
        self._L.tds_b200_get_dims(self._h, dims)
        (self.n_envs, self.n_stride, self.n_q, self.n_qd, self.n_tau, self.n_links,
         self.n_contact_points, self.n_act) = list(dims)
        self.device = device
        self.param_ids = []   # installed physical parameters (set_physical_params)
        self.set_params(dt, gravity, friction, restitution, erp, cfm, pgs_iterations, keep_all_points)
        self.set_precision(precision)

    def close(self):
        if getattr(self, "_h", None):
            self._L.tds_b200_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc, what):
        if rc:
            raise RuntimeError(f"{what} failed (rc={rc}): {_lib.last_error()}")

    def _tangents(self, tangents, what="tangent", names="tangents"):
        """Tangents of a host JVP, pairs (x [n_envs, dim, m] or [n_envs, dim] or None, dim), as contiguous float64 [n_envs, dim, m]
        arrays (None stays None): (arrays, m, single), m = 0 when none is given, single when the first given one is [n_envs, dim]."""
        arrays = []
        for x, dim in tangents:
            if x is not None:
                x = np.asarray(x, dtype=np.float64)
                if x.ndim == 2:
                    x = x[:, :, None]
                if x.shape[:2] != (self.n_envs, dim):
                    raise ValueError(f"{what}: [n_envs, {dim}, m] or [n_envs, {dim}] expected, got {x.shape}")
                x = np.ascontiguousarray(x)
            arrays.append(x)
        ms = {x.shape[2] for x in arrays if x is not None}
        if len(ms) > 1:
            raise ValueError(f"{names}: the same number of tangents m expected")
        first = next((x for x, _ in tangents if x is not None), None)
        return arrays, (ms.pop() if ms else 0), first is not None and np.ndim(first) == 2

    def set_params(self, dt=1e-3, gravity=(0.0, 0.0, -9.81), friction=0.5, restitution=0.0, erp=0.2, cfm=1e-5,
                   pgs_iterations=1, keep_all_points=False):
        g = np.asarray(gravity, dtype=np.float64)
        self.dt = dt
        self._check(self._L.tds_b200_set_params(self._h, dt, _dp(g), friction, restitution, erp, cfm,
                                                pgs_iterations, int(keep_all_points)), "set_params")

    def set_contact_model(self, contact_model=1, spring_k=50000.0, damper_d=5000.0, exponent_n=1.5, v_transition=0.01,
                          hard_contact_condition=True):
        """0: LCP / PGS (reference solver); 1: spring-damper law (parity unpinned, see include/tds_b200.h)."""
        self._check(self._L.tds_b200_set_contact_model(self._h, int(contact_model), spring_k, damper_d, exponent_n, v_transition,
                                                       int(hard_contact_condition)), "set_contact_model")

    def set_env(self, initial_poses, start_link=0, kp=0.0, kd=0.0, max_force=0.0, action_limit=0.4,
                reward_kind=0):
        ip = np.ascontiguousarray(initial_poses, dtype=np.float64)
        self._check(self._L.tds_b200_set_env(self._h, ip.size, _dp(ip), start_link, kp, kd, max_force,
                                             action_limit, reward_kind), "set_env")
        self.n_act = ip.size

    def set_auto_reset(self, enable, reset_q=None):
        rq = None if reset_q is None else np.ascontiguousarray(reset_q, dtype=np.float64)
        if rq is not None:
            assert rq.size == self.n_q
        self._check(self._L.tds_b200_set_auto_reset(self._h, int(enable), _dp(rq)), "set_auto_reset")

    def kernel_name(self):
        """Step kernel launched by the last step call (after the library's selection / fallbacks)."""
        return self._L.tds_b200_kernel_name(self._h).decode()

    def set_precision(self, precision):
        self._check(self._L.tds_b200_set_precision(self._h, precision), "set_precision")

    @property
    def precision(self):
        """The arithmetic selector that runs (PREC_AUTO resolved: mixed for a compiled model, else fp64)."""
        return self._L.tds_b200_get_precision(self._h)

    # ---- device-resident fast path (torch CUDA tensors, SoA [dim, n_stride] float32) ----
    def alloc(self, dim):
        import torch
        return torch.zeros((max(dim, 1), self.n_stride), dtype=torch.float32, device=f"cuda:{self.device}")

    def step_device(self, mode, q, qd, tau_or_action=None, q_out=None, qd_out=None, qdd_out=None, reward=None,
                    done=None, contact_dist=None, link_xf=None, use_pd=False, stream=None):
        q_out = q if q_out is None else q_out
        qd_out = qd if qd_out is None else qd_out
        st = _stream(stream)
        rc = self._L.tds_b200_step_device(self._h, mode, int(use_pd), _ptr(q), _ptr(qd), _ptr(tau_or_action),
                                          _ptr(q_out), _ptr(qd_out), _ptr(qdd_out), _ptr(reward), _ptr(done),
                                          _ptr(contact_dist), _ptr(link_xf), st)
        self._check(rc, "step_device")

    # ---- host-buffer path: numpy [n_envs, dim] float64 in / out ----
    def step_host(self, mode, q, qd, tau_or_action=None, use_pd=False, want_contacts=False):
        q = np.ascontiguousarray(q, dtype=np.float64)
        qd = np.ascontiguousarray(qd, dtype=np.float64)
        n = self.n_envs
        assert q.shape == (n, self.n_q) and qd.shape == (n, self.n_qd)
        t = None
        if tau_or_action is not None:
            t = np.ascontiguousarray(tau_or_action, dtype=np.float64)
            assert t.shape == (n, self.n_act if use_pd else self.n_tau), t.shape
        out = dict(q=np.zeros_like(q), qd=np.zeros_like(qd))
        qdd = np.zeros_like(qd) if mode == MODE_FD else None
        cd = np.zeros((n, max(self.n_contact_points, 1))) if want_contacts else None
        rc = self._L.tds_b200_step_host(self._h, mode, int(use_pd), _dp(q), _dp(qd), _dp(t), _dp(out["q"]),
                                        _dp(out["qd"]), _dp(qdd), _dp(cd))
        self._check(rc, "step_host")
        if qdd is not None:
            out["qdd"] = qdd
        if cd is not None:
            out["contact_dist"] = cd[:, :self.n_contact_points]
            # the contact-pair index list the constraint solver keeps in this step (computed on the device)
            cnt = np.zeros(n, dtype=np.int32)
            links = np.full((n, max(self.n_contact_points, 1), 2), -9, dtype=np.int32)
            self._check(self._L.tds_b200_contact_list_host(self._h, ctypes.c_void_p(cnt.ctypes.data),
                                                           ctypes.c_void_p(links.ctypes.data)), "contact_list_host")
            out["contact_count"] = cnt
            out["contact_links"] = links[:, :self.n_contact_points]
            # ... and which candidates (rows of contact_pairs()) they are: needed to tell the multibodies of a world apart
            cand = np.full((n, max(self.n_contact_points, 1)), -9, dtype=np.int32)
            self._check(self._L.tds_b200_contact_list_candidates_host(self._h, ctypes.c_void_p(cnt.ctypes.data),
                                                                      ctypes.c_void_p(cand.ctypes.data)), "contact_list_candidates_host")
            out["contact_candidates"] = cand[:, :self.n_contact_points]
        return out

    def step_jacobian_host(self, mode, q, qd, tau_or_action=None, use_pd=False):
        """Dense Jacobian of one step per environment (forward-mode dual numbers on the GPU): [n, rows, cols] float64,
        rows = q' | qd' (qdd for MODE_FD), cols = q | qd | tau, or q | qd | action | kp, kd, max_force with use_pd."""
        q = np.ascontiguousarray(q, dtype=np.float64)
        qd = np.ascontiguousarray(qd, dtype=np.float64)
        t = None if tau_or_action is None else np.ascontiguousarray(tau_or_action, dtype=np.float64)
        dims = (ctypes.c_int * 2)()
        self._check(self._L.tds_b200_jacobian_dims(self._h, mode, int(use_pd), dims), "jacobian_dims")
        jac = np.zeros((self.n_envs, dims[0], dims[1]))
        self._check(self._L.tds_b200_step_jacobian_host(self._h, mode, int(use_pd), _dp(q), _dp(qd), _dp(t), _dp(jac)), "step_jacobian_host")
        return jac

    def jacobian_dims(self, mode, use_pd=False):
        """(rows, cols) of the step's Jacobian and of its vector-Jacobian product."""
        dims = (ctypes.c_int * 2)()
        self._check(self._L.tds_b200_jacobian_dims(self._h, mode, int(use_pd), dims), "jacobian_dims")
        return dims[0], dims[1]

    def step_vjp_host(self, mode, q, qd, tau_or_action, g_out, use_pd=False):
        """Vector-Jacobian product of one step per environment by reverse mode on the GPU: g_in [n, cols] = g_out [n, rows]^T J,
        rows / cols as in step_jacobian_host.  The gradient is that of the fp64 world-frame step at the fp32-rounded inputs, of the
        branch taken (contact set, clamps)."""
        q = np.ascontiguousarray(q, dtype=np.float64)
        qd = np.ascontiguousarray(qd, dtype=np.float64)
        t = None if tau_or_action is None else np.ascontiguousarray(tau_or_action, dtype=np.float64)
        rows, cols = self.jacobian_dims(mode, use_pd)
        g = np.ascontiguousarray(g_out, dtype=np.float64)
        assert g.shape == (self.n_envs, rows), (g.shape, rows)
        g_in = np.zeros((self.n_envs, cols))
        self._check(self._L.tds_b200_step_vjp_host(self._h, mode, int(use_pd), _dp(q), _dp(qd), _dp(t), _dp(g), _dp(g_in)), "step_vjp_host")
        return g_in

    def step_vjp_device(self, mode, q, qd, tau_or_action, g_out, g_in, use_pd=False, stream=None):
        """Device version of step_vjp_host on the SoA layout: q, qd, tau_or_action float32 CUDA tensors [dim, n_stride] as for
        step_device, g_out [rows, n_stride] and g_in [cols, n_stride] float64 CUDA tensors.  Synchronises the stream once per chunk
        of environments (see include/tds_b200.h)."""
        st = _stream(stream)
        self._check(self._L.tds_b200_step_vjp_device(self._h, mode, int(use_pd), _ptr(q), _ptr(qd), _ptr(tau_or_action), _ptr(g_out),
                                                     _ptr(g_in), st), "step_vjp_device")

    # ---- per-environment physical parameters (DESIGN.md section 7.9) ----
    def set_physical_params(self, names_or_ids, values=None):
        """Install physical parameters per environment: names (tds_b200.model.param_names) or ids, and values float64 [n_envs, k]
        or [k] (every environment), a numpy array or a CUDA tensor.  names_or_ids None (or empty) clears the set.  Every stepping
        call then uses each environment's values for these parameters and the model's for the rest."""
        from .model import param_ids
        ids = [] if names_or_ids is None else param_ids(self.model, names_or_ids)
        k = len(ids)
        idv = np.ascontiguousarray(ids, dtype=np.int32)
        idp = ctypes.c_void_p(idv.ctypes.data) if k else None
        if k == 0:
            self._check(self._L.tds_b200_set_physical_params_host(self._h, 0, None, None), "set_physical_params")
        elif hasattr(values, "is_cuda") and values.is_cuda:
            import torch
            v = values.to(torch.float64)
            if v.dim() == 1:
                v = v.unsqueeze(0).expand(self.n_envs, k)
            if tuple(v.shape) != (self.n_envs, k):
                raise ValueError(f"values: [n_envs, {k}] or [{k}] expected, got {tuple(values.shape)}")
            soa = torch.zeros((k, self.n_stride), dtype=torch.float64, device=v.device)
            soa[:, :self.n_envs] = v.t()
            st = torch.cuda.current_stream(v.device)
            self._check(self._L.tds_b200_set_physical_params_device(self._h, k, idp, _ptr(soa), ctypes.c_void_p(st.cuda_stream)),
                        "set_physical_params")
            st.synchronize()   # the simulator's copy is complete before soa is released
        else:
            v = np.asarray(values, dtype=np.float64)
            if v.ndim == 1:
                v = np.broadcast_to(v, (self.n_envs, k))
            if v.shape != (self.n_envs, k):
                raise ValueError(f"values: [n_envs, {k}] or [{k}] expected, got {v.shape}")
            v = np.ascontiguousarray(v)
            self._check(self._L.tds_b200_set_physical_params_host(self._h, k, idp, _dp(v)), "set_physical_params")
        self.param_ids = ids

    def param_count(self):
        """Number of physical parameter ids of the model (include/tds_b200.h)."""
        return self._L.tds_b200_param_count(self._h)

    def step_param_jacobian_host(self, mode, q, qd, tau_or_action=None, use_pd=False):
        """d(outputs) / d(installed parameters) of one step per environment by dual numbers: [n, rows, k] float64, rows as in
        step_jacobian_host, columns in the order of set_physical_params."""
        q = np.ascontiguousarray(q, dtype=np.float64)
        qd = np.ascontiguousarray(qd, dtype=np.float64)
        t = None if tau_or_action is None else np.ascontiguousarray(tau_or_action, dtype=np.float64)
        rows, _ = self.jacobian_dims(mode, use_pd)
        jac = np.zeros((self.n_envs, rows, len(self.param_ids)))
        self._check(self._L.tds_b200_step_param_jacobian_host(self._h, mode, int(use_pd), _dp(q), _dp(qd), _dp(t), _dp(jac)),
                    "step_param_jacobian_host")
        return jac

    def step_vjp_params_host(self, mode, q, qd, tau_or_action, g_out, use_pd=False):
        """step_vjp_host with the installed parameters as further inputs: returns (g_in [n, cols], g_par [n, k])."""
        q = np.ascontiguousarray(q, dtype=np.float64)
        qd = np.ascontiguousarray(qd, dtype=np.float64)
        t = None if tau_or_action is None else np.ascontiguousarray(tau_or_action, dtype=np.float64)
        rows, cols = self.jacobian_dims(mode, use_pd)
        g = np.ascontiguousarray(g_out, dtype=np.float64)
        assert g.shape == (self.n_envs, rows), (g.shape, rows)
        g_in = np.zeros((self.n_envs, cols))
        g_par = np.zeros((self.n_envs, len(self.param_ids)))
        self._check(self._L.tds_b200_step_vjp_params_host(self._h, mode, int(use_pd), _dp(q), _dp(qd), _dp(t), _dp(g), _dp(g_in),
                                                          _dp(g_par)), "step_vjp_params_host")
        return g_in, g_par

    def step_vjp_params_device(self, mode, q, qd, tau_or_action, g_out, g_in, g_par, use_pd=False, stream=None):
        """step_vjp_device with the installed parameters: g_par [k, n_stride] float64 CUDA tensor; g_in may be None."""
        st = _stream(stream)
        self._check(self._L.tds_b200_step_vjp_params_device(self._h, mode, int(use_pd), _ptr(q), _ptr(qd), _ptr(tau_or_action),
                                                            _ptr(g_out), _ptr(g_in), _ptr(g_par), st), "step_vjp_params_device")

    def step_jvp_host(self, mode, q, qd, tau_or_action, t_in, t_par=None, use_pd=False):
        """Jacobian-vector products of one step per environment by forward mode on the GPU: t_out [n, rows, m] = J V for the m
        tangents t_in [n, cols, m] of the inputs (rows / cols as in step_jacobian_host) and t_par [n, k, m] of the installed
        parameters; either may be None.  A tangent given as [n, cols] (or [n, k]) is m = 1, and the result is then [n, rows].
        Same derivative as step_jacobian_host: m = cols identity tangents give the Jacobian."""
        q = np.ascontiguousarray(q, dtype=np.float64)
        qd = np.ascontiguousarray(qd, dtype=np.float64)
        t = None if tau_or_action is None else np.ascontiguousarray(tau_or_action, dtype=np.float64)
        rows, cols = self.jacobian_dims(mode, use_pd)
        (ti, tp), m, single = self._tangents([(t_in, cols), (t_par, len(self.param_ids))], names="t_in and t_par")
        out = np.zeros((self.n_envs, rows, max(m, 1)))
        self._check(self._L.tds_b200_step_jvp_host(self._h, mode, int(use_pd), _dp(q), _dp(qd), _dp(t), m, _dp(ti), _dp(tp), _dp(out)),
                    "step_jvp_host")
        return out[:, :, 0] if single else out

    def step_jvp_device(self, mode, q, qd, tau_or_action, m, t_in, t_par, t_out, use_pd=False, stream=None):
        """Device version of step_jvp_host on the SoA layout: q, qd, tau_or_action float32 CUDA tensors [dim, n_stride] as for
        step_device; t_in [cols * m, n_stride], t_par [k * m, n_stride] (either may be None) and t_out [rows * m, n_stride] float64
        CUDA tensors, entry (c, j) at row c * m + j.  Asynchronous on the stream."""
        st = _stream(stream)
        self._check(self._L.tds_b200_step_jvp_device(self._h, mode, int(use_pd), _ptr(q), _ptr(qd), _ptr(tau_or_action), int(m), _ptr(t_in),
                                                     _ptr(t_par), _ptr(t_out), st), "step_jvp_device")

    # ---- joint-space mass matrix M(q) (DESIGN.md section 7.12) ----
    def mass_matrix_host(self, q):
        """M(q) of every environment: [n, n_qd, n_qd] float64, symmetric, by the CRBA of the world-frame step in fp64 at the
        fp32-rounded q [n, n_q] (qd plays no part).  Installed physical parameters give each environment its own masses, centres of
        mass and inertias.  A world of several multibodies gives the block-diagonal matrix."""
        q = np.ascontiguousarray(q, dtype=np.float64)
        assert q.shape == (self.n_envs, self.n_q), q.shape
        M = np.zeros((self.n_envs, self.n_qd, self.n_qd))
        self._check(self._L.tds_b200_mass_matrix_host(self._h, _dp(q), _dp(M)), "mass_matrix_host")
        return M

    def mass_matrix_device(self, q, M, stream=None):
        """Device version of mass_matrix_host on the SoA layout: q float32 CUDA tensor [n_q, n_stride] as for step_device, M float64
        CUDA tensor [n_qd * n_qd, n_stride], entry (r, c) at row r * n_qd + c.  Asynchronous on the stream."""
        st = _stream(stream)
        self._check(self._L.tds_b200_mass_matrix_device(self._h, _ptr(q), _ptr(M), st), "mass_matrix_device")

    def mass_matrix_jvp_host(self, q, t_q, t_par=None):
        """Directional derivatives of M: dM [n, n_qd, n_qd, m] = sum_c dM/dq_c t_q[c] + sum_s dM/dp_s t_par[s] for the m tangents
        t_q [n, n_q, m] of q and t_par [n, k, m] of the installed parameters (either may be None); a tangent given as [n, n_q] (or
        [n, k]) is m = 1 and the result is then [n, n_qd, n_qd].  Returns (M, dM)."""
        q = np.ascontiguousarray(q, dtype=np.float64)
        (tq, tp), m, single = self._tangents([(t_q, self.n_q), (t_par, len(self.param_ids))], names="t_q and t_par")
        M =np.zeros((self.n_envs, self.n_qd, self.n_qd))
        dM = np.zeros((self.n_envs, self.n_qd, self.n_qd, max(m, 1)))
        self._check(self._L.tds_b200_mass_matrix_jvp_host(self._h, _dp(q), m, _dp(tq), _dp(tp), _dp(M), _dp(dM)), "mass_matrix_jvp_host")
        return M, (dM[..., 0] if single else dM)

    def mass_matrix_jvp_device(self, q, m, t_q, t_par, t_M, M=None, stream=None):
        """Device version of mass_matrix_jvp_host: q float32 [n_q, n_stride]; t_q [n_q * m, n_stride], t_par [k * m, n_stride] (either
        may be None), t_M [n_qd * n_qd * m, n_stride] and M [n_qd * n_qd, n_stride] (or None) float64 CUDA tensors, entry (c, j) at row
        c * m + j.  Asynchronous on the stream."""
        st = _stream(stream)
        self._check(self._L.tds_b200_mass_matrix_jvp_device(self._h, _ptr(q), int(m), _ptr(t_q), _ptr(t_par), _ptr(M), _ptr(t_M), st),
                    "mass_matrix_jvp_device")

    def mass_matrix_vjp_host(self, q, G):
        """Cotangent G [n, n_qd, n_qd] of M -> (g_q [n, n_q], g_par [n, k] or None without installed parameters): g = sum G * dM/dx."""
        q = np.ascontiguousarray(q, dtype=np.float64)
        G = np.ascontiguousarray(G, dtype=np.float64)
        assert G.shape == (self.n_envs, self.n_qd, self.n_qd), G.shape
        k = len(self.param_ids)
        g_q = np.zeros((self.n_envs, self.n_q))
        g_par = np.zeros((self.n_envs, k)) if k else None
        self._check(self._L.tds_b200_mass_matrix_vjp_host(self._h, _dp(q), _dp(G), _dp(g_q), _dp(g_par)), "mass_matrix_vjp_host")
        return g_q, g_par

    def mass_matrix_vjp_device(self, q, G, g_q, g_par=None, stream=None):
        """Device version of mass_matrix_vjp_host: q float32 [n_q, n_stride], G float64 [n_qd * n_qd, n_stride] in M's layout, g_q
        [n_q, n_stride] and g_par [k, n_stride] float64 CUDA tensors (either may be None, not both).  Asynchronous on the stream."""
        st = _stream(stream)
        self._check(self._L.tds_b200_mass_matrix_vjp_device(self._h, _ptr(q), _ptr(G), _ptr(g_q), _ptr(g_par), st), "mass_matrix_vjp_device")

    # ---- inverse dynamics tau = ID(q, qd, qdd) (DESIGN.md section 7.14) ----
    def _inv_in(self, x, dim, what):
        if x is None:
            return None
        x = np.ascontiguousarray(x, dtype=np.float64)
        if x.shape != (self.n_envs, dim):
            raise ValueError(f"{what}: [n_envs, {dim}] expected, got {x.shape}")
        return x

    def inverse_dynamics_host(self, q, qd=None, qdd=None):
        """tau [n, n_qd] float64: the joint forces for which every environment has the accelerations qdd at (q, qd) under the
        simulator's gravity, by the recursive Newton-Euler algorithm in fp64 at the fp32-rounded q [n, n_q], qd, qdd [n, n_qd] (None:
        zero; the bias forces are inverse_dynamics_host(q, qd)).  Fixed base: the inverse of MODE_FD, stiffness and damping terms
        included; floating base: rows 0..5 are the base wrench in the base frame for the base-frame acceleration qdd[0:6] (include/tds_b200.h).
        Installed physical parameters give each environment its own masses, inertias, stiffness and damping."""
        q = self._inv_in(q, self.n_q, "q")
        qd, qdd = self._inv_in(qd, self.n_qd, "qd"), self._inv_in(qdd, self.n_qd, "qdd")
        tau = np.zeros((self.n_envs, self.n_qd))
        self._check(self._L.tds_b200_inverse_dynamics_host(self._h, _dp(q), _dp(qd), _dp(qdd), _dp(tau)), "inverse_dynamics_host")
        return tau

    def inverse_dynamics_device(self, q, qd, qdd, tau, stream=None):
        """Device version of inverse_dynamics_host on the SoA layout: q float32 CUDA tensor [n_q, n_stride], qd and qdd [n_qd, n_stride]
        (either may be None), tau float64 [n_qd, n_stride].  Asynchronous on the stream."""
        st = _stream(stream)
        self._check(self._L.tds_b200_inverse_dynamics_device(self._h, _ptr(q), _ptr(qd), _ptr(qdd), _ptr(tau), st), "inverse_dynamics_device")

    def inverse_dynamics_jvp_host(self, q, qd, qdd, t_q=None, t_qd=None, t_qdd=None, t_par=None):
        """Directional derivatives of tau: dtau [n, n_qd, m] along the m tangents t_q [n, n_q, m], t_qd and t_qdd [n, n_qd, m] and t_par
        [n, k, m] of the installed parameters (each may be None, not all); tangents given as [n, dim] are m = 1 and the result is then
        [n, n_qd].  Returns (tau, dtau)."""
        q = self._inv_in(q, self.n_q, "q")
        qd, qdd = self._inv_in(qd, self.n_qd, "qd"), self._inv_in(qdd, self.n_qd, "qdd")
        if all(t is None for t in (t_q, t_qd, t_qdd, t_par)):
            raise ValueError("at least one tangent is expected")
        ts, m, single = self._tangents([(t_q, self.n_q), (t_qd, self.n_qd), (t_qdd, self.n_qd), (t_par, len(self.param_ids))])
        tau = np.zeros((self.n_envs, self.n_qd))
        dtau = np.zeros((self.n_envs, self.n_qd, m))
        self._check(self._L.tds_b200_inverse_dynamics_jvp_host(self._h, _dp(q), _dp(qd), _dp(qdd), m, *(_dp(t) for t in ts), _dp(tau),
                                                               _dp(dtau)), "inverse_dynamics_jvp_host")
        return tau, (dtau[..., 0] if single else dtau)

    def inverse_dynamics_jvp_device(self, q, qd, qdd, m, t_q, t_qd, t_qdd, t_par, t_tau, tau=None, stream=None):
        """Device version of inverse_dynamics_jvp_host: q float32 [n_q, n_stride], qd and qdd [n_qd, n_stride] (or None); t_q
        [n_q * m, n_stride], t_qd and t_qdd [n_qd * m, n_stride], t_par [k * m, n_stride] (each may be None, not all), t_tau
        [n_qd * m, n_stride] and tau [n_qd, n_stride] (or None) float64 CUDA tensors, entry (c, j) at row c * m + j.  Asynchronous."""
        st = _stream(stream)
        self._check(self._L.tds_b200_inverse_dynamics_jvp_device(self._h, _ptr(q), _ptr(qd), _ptr(qdd), int(m), _ptr(t_q), _ptr(t_qd),
                                                                 _ptr(t_qdd), _ptr(t_par), _ptr(tau), _ptr(t_tau), st),
                    "inverse_dynamics_jvp_device")

    def inverse_dynamics_vjp_host(self, q, qd, qdd, G):
        """Cotangent G [n, n_qd] of tau -> (g_q [n, n_q], g_qd [n, n_qd], g_qdd [n, n_qd], g_par [n, k] or None without installed
        parameters): g_x = sum_r G[r] dtau[r]/dx."""
        q = self._inv_in(q, self.n_q, "q")
        qd, qdd = self._inv_in(qd, self.n_qd, "qd"), self._inv_in(qdd, self.n_qd, "qdd")
        G = self._inv_in(G, self.n_qd, "G")
        k = len(self.param_ids)
        g_q, g_qd, g_qdd = np.zeros((self.n_envs, self.n_q)), np.zeros((self.n_envs, self.n_qd)), np.zeros((self.n_envs, self.n_qd))
        g_par = np.zeros((self.n_envs, k)) if k else None
        self._check(self._L.tds_b200_inverse_dynamics_vjp_host(self._h, _dp(q), _dp(qd), _dp(qdd), _dp(G), _dp(g_q), _dp(g_qd), _dp(g_qdd),
                                                               _dp(g_par)), "inverse_dynamics_vjp_host")
        return g_q, g_qd, g_qdd, g_par

    def inverse_dynamics_vjp_device(self, q, qd, qdd, G, g_q, g_qd, g_qdd, g_par=None, stream=None):
        """Device version of inverse_dynamics_vjp_host: q float32 [n_q, n_stride], qd and qdd [n_qd, n_stride] (or None), G float64
        [n_qd, n_stride], g_q [n_q, n_stride], g_qd and g_qdd [n_qd, n_stride], g_par [k, n_stride] float64 CUDA tensors (each may be
        None, not all).  Asynchronous on the stream."""
        st = _stream(stream)
        self._check(self._L.tds_b200_inverse_dynamics_vjp_device(self._h, _ptr(q), _ptr(qd), _ptr(qdd), _ptr(G), _ptr(g_q), _ptr(g_qd),
                                                                 _ptr(g_qdd), _ptr(g_par), st), "inverse_dynamics_vjp_device")

    # ---- derivatives of the inverse dynamics (DESIGN.md section 7.23) ----
    def inverse_dynamics_derivatives_host(self, q, qd=None, qdd=None):
        """(dtau_dq, dtau_dqd) [n, n_qd, n_qd] float64: the derivatives of inverse_dynamics_host's tau at the fp32-rounded q [n, n_q], qd,
        qdd [n, n_qd] (None: zero), row r = tau_r, column c = a tangent direction in M's coordinates: column k of dtau_dq is the
        derivative along the motion with velocity e_k, i.e. inverse_dynamics_jvp_host along t_q = dq_dt(q, e_k) (include/tds_b200.h).
        dtau / dqdd is mass_matrix_host(q)."""
        q = self._inv_in(q, self.n_q, "q")
        qd, qdd = self._inv_in(qd, self.n_qd, "qd"), self._inv_in(qdd, self.n_qd, "qdd")
        a, b = np.zeros((self.n_envs, self.n_qd, self.n_qd)), np.zeros((self.n_envs, self.n_qd, self.n_qd))
        self._check(self._L.tds_b200_inverse_dynamics_derivatives_host(self._h, _dp(q), _dp(qd), _dp(qdd), _dp(a), _dp(b)),
                    "inverse_dynamics_derivatives_host")
        return a, b

    def inverse_dynamics_derivatives_device(self, q, qd, qdd, dtau_dq, dtau_dqd, stream=None):
        """Device version of inverse_dynamics_derivatives_host on the SoA layout: q float32 CUDA tensor [n_q, n_stride], qd and qdd
        [n_qd, n_stride] (either may be None), dtau_dq and dtau_dqd float64 [n_qd * n_qd, n_stride] (either may be None, not both).
        Asynchronous on the stream."""
        st = _stream(stream)
        self._check(self._L.tds_b200_inverse_dynamics_derivatives_device(self._h, _ptr(q), _ptr(qd), _ptr(qdd), _ptr(dtau_dq), _ptr(dtau_dqd),
                                                                         st), "inverse_dynamics_derivatives_device")

    def inverse_dynamics_derivatives_jvp_host(self, q, qd, qdd, t_q=None, t_qd=None, t_qdd=None, t_par=None):
        """Directional derivatives of (dtau_dq, dtau_dqd): each [n, n_qd, n_qd, m] along the m tangents t_q [n, n_q, m], t_qd and t_qdd
        [n, n_qd, m] and t_par [n, k, m] (each may be None, not all; [n, dim] is m = 1 and gives [n, n_qd, n_qd]).  Returns (dtau_dq,
        dtau_dqd, t_dtau_dq, t_dtau_dqd)."""
        q = self._inv_in(q, self.n_q, "q")
        qd, qdd = self._inv_in(qd, self.n_qd, "qd"), self._inv_in(qdd, self.n_qd, "qdd")
        if all(t is None for t in (t_q, t_qd, t_qdd, t_par)):
            raise ValueError("at least one tangent is expected")
        ts, m, single = self._tangents([(t_q, self.n_q), (t_qd, self.n_qd), (t_qdd, self.n_qd), (t_par, len(self.param_ids))])
        nd = self.n_qd
        a, b = np.zeros((self.n_envs, nd, nd)), np.zeros((self.n_envs, nd, nd))
        ta, tb = np.zeros((self.n_envs, nd, nd, m)), np.zeros((self.n_envs, nd, nd, m))
        self._check(self._L.tds_b200_inverse_dynamics_derivatives_jvp_host(self._h, _dp(q), _dp(qd), _dp(qdd), m, *(_dp(t) for t in ts),
                                                                           _dp(a), _dp(b), _dp(ta), _dp(tb)),
                    "inverse_dynamics_derivatives_jvp_host")
        return (a, b, ta[..., 0], tb[..., 0]) if single else (a, b, ta, tb)

    def inverse_dynamics_derivatives_jvp_device(self, q, qd, qdd, m, t_q, t_qd, t_qdd, t_par, t_dtau_dq, t_dtau_dqd, dtau_dq=None,
                                                dtau_dqd=None, stream=None):
        """Device version of inverse_dynamics_derivatives_jvp_host: q float32 [n_q, n_stride], qd and qdd [n_qd, n_stride] (or None);
        t_q [n_q * m, n_stride], t_qd and t_qdd [n_qd * m, n_stride], t_par [k * m, n_stride] (each may be None, not all), t_dtau_dq and
        t_dtau_dqd [n_qd * n_qd * m, n_stride] (either may be None, not both) and the values [n_qd * n_qd, n_stride] (or None) float64
        CUDA tensors, entry (c, j) at row c * m + j.  Asynchronous."""
        st = _stream(stream)
        self._check(self._L.tds_b200_inverse_dynamics_derivatives_jvp_device(
            self._h, _ptr(q), _ptr(qd), _ptr(qdd), int(m), _ptr(t_q), _ptr(t_qd), _ptr(t_qdd), _ptr(t_par), _ptr(dtau_dq), _ptr(dtau_dqd),
            _ptr(t_dtau_dq), _ptr(t_dtau_dqd), st), "inverse_dynamics_derivatives_jvp_device")

    def inverse_dynamics_derivatives_vjp_host(self, q, qd, qdd, G_dq=None, G_dqd=None):
        """Cotangents G_dq, G_dqd [n, n_qd, n_qd] of (dtau_dq, dtau_dqd) (either may be None, not both) -> (g_q [n, n_q], g_qd [n, n_qd],
        g_qdd [n, n_qd], g_par [n, k] or None without installed parameters)."""
        q = self._inv_in(q, self.n_q, "q")
        qd, qdd = self._inv_in(qd, self.n_qd, "qd"), self._inv_in(qdd, self.n_qd, "qdd")
        nn = self.n_qd * self.n_qd
        G_dq = None if G_dq is None else self._inv_in(np.reshape(G_dq, (self.n_envs, nn)), nn, "G_dq")
        G_dqd = None if G_dqd is None else self._inv_in(np.reshape(G_dqd, (self.n_envs, nn)), nn, "G_dqd")
        k = len(self.param_ids)
        g_q, g_qd, g_qdd = np.zeros((self.n_envs, self.n_q)), np.zeros((self.n_envs, self.n_qd)), np.zeros((self.n_envs, self.n_qd))
        g_par = np.zeros((self.n_envs, k)) if k else None
        self._check(self._L.tds_b200_inverse_dynamics_derivatives_vjp_host(self._h, _dp(q), _dp(qd), _dp(qdd), _dp(G_dq), _dp(G_dqd), _dp(g_q),
                                                                           _dp(g_qd), _dp(g_qdd), _dp(g_par)),
                    "inverse_dynamics_derivatives_vjp_host")
        return g_q, g_qd, g_qdd, g_par

    def inverse_dynamics_derivatives_vjp_device(self, q, qd, qdd, G_dq, G_dqd, g_q, g_qd, g_qdd, g_par=None, stream=None):
        """Device version of inverse_dynamics_derivatives_vjp_host: q float32 [n_q, n_stride], qd and qdd [n_qd, n_stride] (or None),
        G_dq and G_dqd float64 [n_qd * n_qd, n_stride] (either may be None, not both), g_q [n_q, n_stride], g_qd and g_qdd [n_qd,
        n_stride], g_par [k, n_stride] float64 CUDA tensors (each may be None, not all).  Asynchronous on the stream."""
        st = _stream(stream)
        self._check(self._L.tds_b200_inverse_dynamics_derivatives_vjp_device(self._h, _ptr(q), _ptr(qd), _ptr(qdd), _ptr(G_dq), _ptr(G_dqd),
                                                                             _ptr(g_q), _ptr(g_qd), _ptr(g_qdd), _ptr(g_par), st),
                    "inverse_dynamics_derivatives_vjp_device")

    # ---- centre of mass, centroidal momentum matrix and its bias (DESIGN.md section 7.16) ----
    def centroidal_host(self, q, qd=None):
        """(m [n], c [n, 3], I_G [n, 3, 3], A [n, 6, n_qd], bias [n, 6]) float64 at the fp32-rounded q [n, n_q] and qd [n, n_qd] (None:
        zero): the total mass of the links and a floating base, their centre of mass c in world coordinates and rotational inertia about c
        in world axes, the centroidal momentum matrix A_G (rows [angular momentum about c; linear momentum] in world axes, columns in
        the coordinates of the mass matrix: h_G = A qd) and its bias A_G' qd (the rate of h_G at qdd = 0, velocity terms only).
        Installed masses, centres of mass and inertias apply per environment (include/tds_b200.h)."""
        q = self._inv_in(q, self.n_q, "q")
        qd = self._inv_in(qd, self.n_qd, "qd")
        com, A, bias = np.zeros((self.n_envs, 10)), np.zeros((self.n_envs, 6, self.n_qd)), np.zeros((self.n_envs, 6))
        self._check(self._L.tds_b200_centroidal_host(self._h, _dp(q), _dp(qd), _dp(com), _dp(A), _dp(bias)), "centroidal_host")
        return com[:, 0], com[:, 1:4], _sym3(com[:, 4:10]), A, bias

    def centroidal_device(self, q, qd, com, A, bias, stream=None):
        """Device version of centroidal_host on the SoA layout: q float32 CUDA tensor [n_q, n_stride], qd [n_qd, n_stride] (or None); com
        [10, n_stride] (m, c, I_G xx xy xz yy yz zz), A [6 n_qd, n_stride], bias [6, n_stride] float64 (each may be None, not all).
        Asynchronous on the stream."""
        st = _stream(stream)
        self._check(self._L.tds_b200_centroidal_device(self._h, _ptr(q), _ptr(qd), _ptr(com), _ptr(A), _ptr(bias), st), "centroidal_device")

    def centroidal_jvp_host(self, q, qd=None, t_q=None, t_qd=None, t_par=None):
        """Directional derivatives (dcom [n, 10, m], dA [n, 6, n_qd, m], dbias [n, 6, m]) of the outputs of centroidal_host in its
        com-record layout (m, c, I_G xx xy xz yy yz zz) along m tangents t_q [n, n_q, m], t_qd [n, n_qd, m] and t_par [n, k, m] (each may
        be None, not all); tangents given as [n, dim] are m = 1 and drop the last axis."""
        q = self._inv_in(q, self.n_q, "q")
        qd = self._inv_in(qd, self.n_qd, "qd")
        if all(t is None for t in (t_q, t_qd, t_par)):
            raise ValueError("at least one tangent is expected")
        ts, m, single = self._tangents([(t_q, self.n_q), (t_qd, self.n_qd), (t_par, len(self.param_ids))])
        n = self.n_envs
        dcom, dA, dbias = np.zeros((n, 10, m)), np.zeros((n, 6, self.n_qd, m)), np.zeros((n, 6, m))
        self._check(self._L.tds_b200_centroidal_jvp_host(self._h, _dp(q), _dp(qd), m, *(_dp(t) for t in ts), _dp(dcom), _dp(dA), _dp(dbias)),
                    "centroidal_jvp_host")
        return (dcom[..., 0], dA[..., 0], dbias[..., 0]) if single else (dcom, dA, dbias)

    def centroidal_jvp_device(self, q, qd, m, t_q, t_qd, t_par, t_com, t_A, t_bias, stream=None):
        """Device version of centroidal_jvp_host: q float32 [n_q, n_stride], qd [n_qd, n_stride] (or None); t_q [n_q * m, n_stride], t_qd
        [n_qd * m, n_stride], t_par [k * m, n_stride] (each may be None, not all), t_com [10 m, n_stride], t_A [6 n_qd m, n_stride], t_bias
        [6 m, n_stride] (each may be None, not all) float64 CUDA tensors, entry (r, j) at row r * m + j.  Asynchronous on the stream."""
        st = _stream(stream)
        self._check(self._L.tds_b200_centroidal_jvp_device(self._h, _ptr(q), _ptr(qd), int(m), _ptr(t_q), _ptr(t_qd), _ptr(t_par), _ptr(t_com),
                                                           _ptr(t_A), _ptr(t_bias), st), "centroidal_jvp_device")

    def centroidal_vjp_host(self, q, qd=None, G_com=None, G_A=None, G_bias=None):
        """Cotangents G_com [n, 10] (com-record layout), G_A [n, 6, n_qd], G_bias [n, 6] (None: zero, not all) -> (g_q [n, n_q], g_qd
        [n, n_qd], g_par [n, k] or None without installed parameters)."""
        q = self._inv_in(q, self.n_q, "q")
        qd = self._inv_in(qd, self.n_qd, "qd")
        if G_com is None and G_A is None and G_bias is None:
            raise ValueError("at least one cotangent is expected")
        G_com = self._inv_in(G_com, 10, "G_com")
        G_A = None if G_A is None else self._inv_in(np.reshape(G_A, (self.n_envs, -1)), 6 * self.n_qd, "G_A")
        G_bias = self._inv_in(G_bias, 6, "G_bias")
        k = len(self.param_ids)
        g_q, g_qd = np.zeros((self.n_envs, self.n_q)), np.zeros((self.n_envs, self.n_qd))
        g_par = np.zeros((self.n_envs, k)) if k else None
        self._check(self._L.tds_b200_centroidal_vjp_host(self._h, _dp(q), _dp(qd), _dp(G_com), _dp(G_A), _dp(G_bias), _dp(g_q), _dp(g_qd),
                                                         _dp(g_par)), "centroidal_vjp_host")
        return g_q, g_qd, g_par

    def centroidal_vjp_device(self, q, qd, G_com, G_A, G_bias, g_q, g_qd, g_par=None, stream=None):
        """Device version of centroidal_vjp_host: q float32 [n_q, n_stride], qd [n_qd, n_stride] (or None), G_com [10, n_stride], G_A
        [6 n_qd, n_stride], G_bias [6, n_stride] (each may be None, not all), g_q [n_q, n_stride], g_qd [n_qd, n_stride], g_par [k, n_stride]
        float64 CUDA tensors (each may be None, not all).  Asynchronous on the stream."""
        st = _stream(stream)
        self._check(self._L.tds_b200_centroidal_vjp_device(self._h, _ptr(q), _ptr(qd), _ptr(G_com), _ptr(G_A), _ptr(G_bias), _ptr(g_q),
                                                           _ptr(g_qd), _ptr(g_par), st), "centroidal_vjp_device")

    # ---- the step with its contact records (DESIGN.md section 7.15) ----
    def contact_rows(self, mode=MODE_FULL, use_pd=False):
        """(rows, cols) of the derivatives of step_contacts: rows q' | qd' | records (n_q + n_qd + 10 n_contact_points), cols as in
        step_jacobian_host."""
        rows, cols = self.jacobian_dims(mode, use_pd)
        return rows + 10 * self.n_contact_points, cols

    def _step_args(self, q, qd, tau_or_action):
        q = np.ascontiguousarray(q, dtype=np.float64)
        qd = np.ascontiguousarray(qd, dtype=np.float64)
        if q.shape != (self.n_envs, self.n_q) or qd.shape != (self.n_envs, self.n_qd):
            raise ValueError(f"q [n_envs, {self.n_q}] and qd [n_envs, {self.n_qd}] expected, got {q.shape} and {qd.shape}")
        t = None if tau_or_action is None else np.ascontiguousarray(tau_or_action, dtype=np.float64)
        return q, qd, t

    def step_contacts_host(self, mode, q, qd, tau_or_action=None, use_pd=False):
        """One step (MODE_FULL or MODE_WORLD) on the world-frame kernel that also reports its contacts: (q' [n, n_q], qd' [n, n_qd],
        C [n, n_contact_points, 10] float64), a record per contact candidate: normal on b [3], point on b [3], distance, impulse on
        body b [3] (N s) at the point on b, world coordinates (include/tds_b200.h).  q' and qd' are bitwise those of step_device on
        the world-frame kernel."""
        q, qd, t = self._step_args(q, qd, tau_or_action)
        qo, qdo = np.zeros_like(q), np.zeros_like(qd)
        C = np.zeros((self.n_envs, max(self.n_contact_points, 1), 10))
        self._check(self._L.tds_b200_step_contacts_host(self._h, mode, int(use_pd), _dp(q), _dp(qd), _dp(t), _dp(qo), _dp(qdo), _dp(C)),
                    "step_contacts_host")
        return qo, qdo, C[:, :self.n_contact_points]

    def step_contacts_device(self, mode, q, qd, tau_or_action, q_out, qd_out, contacts, use_pd=False, stream=None):
        """Device version of step_contacts_host on the SoA layout: q, qd, tau_or_action, q_out, qd_out float32 CUDA tensors
        [dim, n_stride] as for step_device, contacts float32 [10 * n_contact_points, n_stride] (row r of candidate k at 10 k + r).
        Asynchronous on the stream."""
        st = _stream(stream)
        self._check(self._L.tds_b200_step_contacts_device(self._h, mode, int(use_pd), _ptr(q), _ptr(qd), _ptr(tau_or_action), _ptr(q_out),
                                                          _ptr(qd_out), _ptr(contacts), st), "step_contacts_device")

    def step_contacts_jvp_host(self, mode, q, qd, tau_or_action, t_in, t_par=None, use_pd=False):
        """step_jvp_host of step_contacts: t_out [n, rows, m] with rows q' | qd' | records (contact_rows), MODE_FULL."""
        q, qd, t = self._step_args(q, qd, tau_or_action)
        rows, cols = self.contact_rows(mode, use_pd)
        (ti, tp), m, single = self._tangents([(t_in, cols), (t_par, len(self.param_ids))], names="t_in and t_par")
        out = np.zeros((self.n_envs, rows, max(m, 1)))
        self._check(self._L.tds_b200_step_contacts_jvp_host(self._h, mode, int(use_pd), _dp(q), _dp(qd), _dp(t), m, _dp(ti), _dp(tp),
                                                            _dp(out)), "step_contacts_jvp_host")
        return out[:, :, 0] if single else out

    def step_contacts_jvp_device(self, mode, q, qd, tau_or_action, m, t_in, t_par, t_out, use_pd=False, stream=None):
        """Device version of step_contacts_jvp_host, layouts as step_jvp_device with t_out [rows * m, n_stride] (contact_rows)."""
        st = _stream(stream)
        self._check(self._L.tds_b200_step_contacts_jvp_device(self._h, mode, int(use_pd), _ptr(q), _ptr(qd), _ptr(tau_or_action), int(m),
                                                              _ptr(t_in), _ptr(t_par), _ptr(t_out), st), "step_contacts_jvp_device")

    def step_contacts_vjp_host(self, mode, q, qd, tau_or_action, g_out, use_pd=False):
        """Vector-Jacobian product of step_contacts (MODE_FULL): g_out [n, rows] over q' | qd' | records (contact_rows) -> (g_in
        [n, cols], g_par [n, k] or None without installed parameters)."""
        q, qd, t = self._step_args(q, qd, tau_or_action)
        rows, cols = self.contact_rows(mode, use_pd)
        g = np.ascontiguousarray(g_out, dtype=np.float64)
        if g.shape != (self.n_envs, rows):
            raise ValueError(f"g_out: [n_envs, {rows}] expected, got {g.shape}")
        g_in = np.zeros((self.n_envs, cols))
        g_par = np.zeros((self.n_envs, len(self.param_ids))) if self.param_ids else None
        self._check(self._L.tds_b200_step_contacts_vjp_host(self._h, mode, int(use_pd), _dp(q), _dp(qd), _dp(t), _dp(g), _dp(g_in),
                                                            _dp(g_par)), "step_contacts_vjp_host")
        return g_in, g_par

    def step_contacts_vjp_device(self, mode, q, qd, tau_or_action, g_out, g_in, g_par=None, use_pd=False, stream=None):
        """Device version of step_contacts_vjp_host: g_out [rows, n_stride], g_in [cols, n_stride], g_par [k, n_stride] float64 CUDA
        tensors (g_in or g_par may be None, not both).  Asynchronous on the stream."""
        st = _stream(stream)
        self._check(self._L.tds_b200_step_contacts_vjp_device(self._h, mode, int(use_pd), _ptr(q), _ptr(qd), _ptr(tau_or_action),
                                                              _ptr(g_out), _ptr(g_in), _ptr(g_par), st), "step_contacts_vjp_device")

    # ---- the step with external wrenches (DESIGN.md section 7.18) ----
    def _wrench_args(self, links, local, W):
        """The point table and the wrenches W [n_envs, K, 6] (or [K, 6] for every environment) as the host entry points take them."""
        keep, K, lp, cp = self._kin_args(links, local)
        w = np.ascontiguousarray(np.broadcast_to(np.asarray(W, dtype=np.float64), (self.n_envs, K, 6))) if K else None
        return keep, K, lp, cp, w

    def step_wrench_host(self, mode, q, qd, tau_or_action, links, local, W, use_pd=False):
        """One step (MODE_FD, MODE_NOCONTACT or MODE_FULL) on the world-frame kernel with a wrench W[e, k] = [n; f] (world axes, rounded to
        fp32) at every point of the table links [K] (-1: the base) / local [K, 3]: (q' [n, n_q], qd' [n, n_qd]), or qdd [n, n_qd] in
        MODE_FD.  The force f acts along a line through the point, n is a pure moment; the generalised force is J^T W with J the 6-row
        point Jacobian of point_motion_host (include/tds_b200.h).  K = 0 is the world-frame step."""
        q, qd, t = self._step_args(q, qd, tau_or_action)
        keep, K, lp, cp, w = self._wrench_args(links, local, W)
        qo, qdo, qddo = np.zeros_like(q), np.zeros_like(qd), np.zeros_like(qd)
        self._check(self._L.tds_b200_step_wrench_host(self._h, mode, int(use_pd), _dp(q), _dp(qd), _dp(t), K, lp, cp, _dp(w), _dp(qo),
                                                      _dp(qdo), _dp(qddo)), "step_wrench_host")
        return qddo if mode == MODE_FD else (qo, qdo)

    def step_wrench_device(self, mode, q, qd, tau_or_action, links, local, W, q_out=None, qd_out=None, qdd_out=None, use_pd=False,
                           stream=None):
        """Device version of step_wrench_host on the SoA layout: q, qd, tau_or_action float32 CUDA tensors [dim, n_stride] as for
        step_device, W float32 [6K, n_stride] (row 6k + r: component r of [n; f] of point k); q_out, qd_out (MODE_NOCONTACT, MODE_FULL)
        or qdd_out (MODE_FD) float32 [dim, n_stride].  The point table is host data.  Asynchronous on the stream."""
        st = _stream(stream)
        keep, K, lp, cp = self._kin_args(links, local)
        self._check(self._L.tds_b200_step_wrench_device(self._h, mode, int(use_pd), _ptr(q), _ptr(qd), _ptr(tau_or_action), K, lp, cp,
                                                        _ptr(W), _ptr(q_out), _ptr(qd_out), _ptr(qdd_out), st), "step_wrench_device")

    def step_wrench_jvp_host(self, mode, q, qd, tau_or_action, links, local, W, t_in=None, t_W=None, t_par=None, use_pd=False):
        """Directional derivatives t_out [n, rows, m] of step_wrench_host (rows q' | qd', or qdd in MODE_FD, as step_jacobian_host)
        along m tangents t_in [n, cols, m] of the step's inputs, t_W [n, K, 6, m] of the wrenches and t_par [n, k, m] of the installed
        parameters (each may be None, not all three); tangents given without the last axis are m = 1 and drop it."""
        q, qd, t = self._step_args(q, qd, tau_or_action)
        keep, K, lp, cp, w = self._wrench_args(links, local, W)
        rows, cols = self.jacobian_dims(mode, use_pd)
        tw = None if t_W is None else np.asarray(t_W, dtype=np.float64)
        single_w = tw is not None and tw.ndim == 3
        if tw is not None:
            tw = tw.reshape(self.n_envs, 6 * K, -1) if not single_w else tw.reshape(self.n_envs, 6 * K)
        (ti, tww, tp), m, single = self._tangents([(t_in, cols), (tw, 6 * K), (t_par, len(self.param_ids))], names="t_in, t_W and t_par")
        if m == 0:
            raise ValueError("at least one tangent is expected")
        out = np.zeros((self.n_envs, rows, m))
        self._check(self._L.tds_b200_step_wrench_jvp_host(self._h, mode, int(use_pd), _dp(q), _dp(qd), _dp(t), K, lp, cp, _dp(w), m, _dp(ti),
                                                          _dp(tww), _dp(tp), _dp(out)), "step_wrench_jvp_host")
        return out[:, :, 0] if single else out

    def step_wrench_jvp_device(self, mode, q, qd, tau_or_action, links, local, W, m, t_in, t_W, t_par, t_out, use_pd=False, stream=None):
        """Device version of step_wrench_jvp_host, layouts as step_jvp_device with t_W [6K * m, n_stride] float64 (entry (6k + r, j) at
        row (6k + r) * m + j); t_in, t_W and t_par may be None, not all three.  Asynchronous on the stream."""
        st = _stream(stream)
        keep, K, lp, cp = self._kin_args(links, local)
        self._check(self._L.tds_b200_step_wrench_jvp_device(self._h, mode, int(use_pd), _ptr(q), _ptr(qd), _ptr(tau_or_action), K, lp, cp,
                                                            _ptr(W), int(m), _ptr(t_in), _ptr(t_W), _ptr(t_par), _ptr(t_out), st),
                    "step_wrench_jvp_device")

    def step_wrench_vjp_host(self, mode, q, qd, tau_or_action, links, local, W, g_out, use_pd=False):
        """Vector-Jacobian product of step_wrench_host: g_out [n, rows] -> (g_in [n, cols], g_W [n, K, 6], g_par [n, k] or None without
        installed parameters)."""
        q, qd, t = self._step_args(q, qd, tau_or_action)
        keep, K, lp, cp, w = self._wrench_args(links, local, W)
        rows, cols = self.jacobian_dims(mode, use_pd)
        g = np.ascontiguousarray(g_out, dtype=np.float64)
        if g.shape != (self.n_envs, rows):
            raise ValueError(f"g_out: [n_envs, {rows}] expected, got {g.shape}")
        g_in, g_W = np.zeros((self.n_envs, cols)), np.zeros((self.n_envs, K, 6))
        g_par = np.zeros((self.n_envs, len(self.param_ids))) if self.param_ids else None
        self._check(self._L.tds_b200_step_wrench_vjp_host(self._h, mode, int(use_pd), _dp(q), _dp(qd), _dp(t), K, lp, cp, _dp(w), _dp(g),
                                                          _dp(g_in), _dp(g_W) if K else None, _dp(g_par)), "step_wrench_vjp_host")
        return g_in, g_W, g_par

    def step_wrench_vjp_device(self, mode, q, qd, tau_or_action, links, local, W, g_out, g_in=None, g_W=None, g_par=None, use_pd=False,
                               stream=None):
        """Device version of step_wrench_vjp_host: g_out [rows, n_stride], g_in [cols, n_stride], g_W [6K, n_stride], g_par [k, n_stride]
        float64 CUDA tensors (g_in, g_W or g_par may be None, not all three).  Asynchronous on the stream."""
        st = _stream(stream)
        keep, K, lp, cp = self._kin_args(links, local)
        self._check(self._L.tds_b200_step_wrench_vjp_device(self._h, mode, int(use_pd), _ptr(q), _ptr(qd), _ptr(tau_or_action), K, lp, cp,
                                                            _ptr(W), _ptr(g_out), _ptr(g_in), _ptr(g_W), _ptr(g_par), st),
                    "step_wrench_vjp_device")

    # ---- forward kinematics and linear point Jacobians (DESIGN.md section 7.13) ----
    @staticmethod
    def _points(links, local):
        """The point table as the C-ABI takes it: (links int32 [K], local float64 [K, 3], K)."""
        lk = np.ascontiguousarray(np.asarray(links, dtype=np.int64).ravel(), dtype=np.int32)
        lc = np.ascontiguousarray(np.asarray(local, dtype=np.float64).reshape(-1, 3))
        if lc.shape[0] != lk.size:
            raise ValueError(f"links [K] and local [K, 3] expected, got {lk.shape} and {lc.shape}")
        return lk, lc, lk.size

    def _kin_args(self, links, local):
        lk, lc, K = self._points(links, local)
        return (lk, lc), K, ctypes.c_void_p(lk.ctypes.data) if K else None, _dp(lc) if K else None

    def kinematics_host(self, q, links, local):
        """Forward kinematics and linear point Jacobians at the fp32-rounded q [n, n_q] (qd plays no part) for the point table links [K]
        (-1: the base) / local [K, 3] (coordinates in the link's frame): (R [n, n_links, 3, 3], p [n, n_links, 3], x [n, K, 3],
        J [n, K, 3, n_qd]), float64, world coordinates.  J follows the reference's point_jacobian (a floating base gives
        [-[x - r0]x^T | I3] with the base's rotation ignored).  Installed physical parameters do not enter."""
        q = np.ascontiguousarray(q, dtype=np.float64)
        assert q.shape == (self.n_envs, self.n_q), q.shape
        keep, K, lp, cp = self._kin_args(links, local)
        xf = np.zeros((self.n_envs, self.n_links, 12))
        x = np.zeros((self.n_envs, K, 3))
        J = np.zeros((self.n_envs, K, 3, self.n_qd))
        self._check(self._L.tds_b200_kinematics_host(self._h, _dp(q), K, lp, cp, _dp(xf), _dp(x), _dp(J)), "kinematics_host")
        return xf[:, :, :9].reshape(self.n_envs, self.n_links, 3, 3), xf[:, :, 9:].copy(), x, J

    def kinematics_device(self, q, links, local, xf=None, x=None, J=None, stream=None):
        """Device version of kinematics_host on the SoA layout: q float32 CUDA tensor [n_q, n_stride]; xf [n_links * 12, n_stride], x [3K,
        n_stride] and J [3K * n_qd, n_stride] float64 CUDA tensors (any may be None, not all three), entry (point k, row r, column c) of J
        at row (3k + r) * n_qd + c.  The point table is host data.  Asynchronous on the stream."""
        st = _stream(stream)
        keep, K, lp, cp = self._kin_args(links, local)
        self._check(self._L.tds_b200_kinematics_device(self._h, _ptr(q), K, lp, cp, _ptr(xf), _ptr(x), _ptr(J), st), "kinematics_device")

    def kinematics_jvp_host(self, q, links, local, t_q):
        """Directional derivatives along m tangents t_q [n, n_q, m] of q: (dxf [n, n_links, 12, m], dx [n, K, 3, m], dJ [n, K, 3, n_qd, m])
        (xf in the layout R row-major | p); a tangent given as [n, n_q] is m = 1 and the trailing axis is dropped."""
        q = np.ascontiguousarray(q, dtype=np.float64)
        (tq,), m, single = self._tangents([(t_q, self.n_q)], what="t_q")
        keep, K, lp, cp = self._kin_args(links, local)
        n = self.n_envs
        dxf, dx, dJ = np.zeros((n, self.n_links, 12, m)), np.zeros((n, K, 3, m)), np.zeros((n, K, 3, self.n_qd, m))
        self._check(self._L.tds_b200_kinematics_jvp_host(self._h, _dp(q), K, lp, cp, m, _dp(tq), _dp(dxf), _dp(dx), _dp(dJ)),
                    "kinematics_jvp_host")
        return (dxf[..., 0], dx[..., 0], dJ[..., 0]) if single else (dxf, dx, dJ)

    def kinematics_jvp_device(self, q, links, local, m, t_q, t_xf=None, t_x=None, t_J=None, stream=None):
        """Device version of kinematics_jvp_host: q float32 [n_q, n_stride]; t_q [n_q * m, n_stride] and t_xf [n_links * 12 * m, n_stride],
        t_x [3K * m, n_stride], t_J [3K * n_qd * m, n_stride] (any may be None, not all three) float64 CUDA tensors, entry (r, j) at row
        r * m + j.  Asynchronous on the stream."""
        st = _stream(stream)
        keep, K, lp, cp = self._kin_args(links, local)
        self._check(self._L.tds_b200_kinematics_jvp_device(self._h, _ptr(q), K, lp, cp, int(m), _ptr(t_q), _ptr(t_xf), _ptr(t_x), _ptr(t_J),
                                                           st), "kinematics_jvp_device")

    def kinematics_vjp_host(self, q, links, local, G_xf=None, G_x=None, G_J=None):
        """Cotangents G_xf [n, n_links, 12], G_x [n, K, 3], G_J [n, K, 3, n_qd] (None: zero, not all three) -> g_q [n, n_q] =
        sum G * d(outputs)/dq."""
        q = np.ascontiguousarray(q, dtype=np.float64)
        keep, K, lp, cp = self._kin_args(links, local)
        n = self.n_envs

        def prep(G, shape):
            if G is None:
                return None
            G = np.ascontiguousarray(G, dtype=np.float64)
            assert G.size == int(np.prod(shape)), (G.shape, shape)
            return G
        gxf, gx, gJ = prep(G_xf, (n, self.n_links, 12)), prep(G_x, (n, K, 3)), prep(G_J, (n, K, 3, self.n_qd))
        g_q = np.zeros((n, self.n_q))
        self._check(self._L.tds_b200_kinematics_vjp_host(self._h, _dp(q), K, lp, cp, _dp(gxf), _dp(gx), _dp(gJ), _dp(g_q)),
                    "kinematics_vjp_host")
        return g_q

    def kinematics_vjp_device(self, q, links, local, G_xf, G_x, G_J, g_q, stream=None):
        """Device version of kinematics_vjp_host: q float32 [n_q, n_stride], cotangents float64 in the layouts of kinematics_device (None:
        zero, not all three), g_q float64 [n_q, n_stride] CUDA tensors.  Asynchronous on the stream."""
        st = _stream(stream)
        keep, K, lp, cp = self._kin_args(links, local)
        self._check(self._L.tds_b200_kinematics_vjp_device(self._h, _ptr(q), K, lp, cp, _ptr(G_xf), _ptr(G_x), _ptr(G_J), _ptr(g_q), st),
                    "kinematics_vjp_device")

    # ---- spatial point Jacobians, point velocities and accelerations (DESIGN.md section 7.17) ----
    def point_motion_host(self, q, qd, links, local, qdd=None):
        """Spatial point Jacobians, velocities and accelerations at the fp32-rounded q [n, n_q], qd and qdd [n, n_qd] (None: zero) for the
        point table of kinematics_host: (J [n, K, 6, n_qd], vel [n, K, 6], acc [n, K, 6]) float64, world axes, rows [w; x'] of the
        point's link angular velocity and the velocity of its world position: vel = J qd, acc = [w'; x''] = J qdd + J' qd.  Columns in
        the coordinates of mass_matrix_host: a floating base's are the base twist's, [R_b | 0; -[x - p_b]x R_b | R_b] - unlike
        kinematics_host, whose base columns ignore the base rotation.  Gravity and installed physical parameters do not enter."""
        q = self._inv_in(q, self.n_q, "q")
        qd, qdd = self._inv_in(qd, self.n_qd, "qd"), self._inv_in(qdd, self.n_qd, "qdd")
        keep, K, lp, cp = self._kin_args(links, local)
        n = self.n_envs
        J, vel, acc = np.zeros((n, K, 6, self.n_qd)), np.zeros((n, K, 6)), np.zeros((n, K, 6))
        self._check(self._L.tds_b200_point_motion_host(self._h, _dp(q), _dp(qd), _dp(qdd), K, lp, cp, _dp(J), _dp(vel), _dp(acc)),
                    "point_motion_host")
        return J, vel, acc

    def point_motion_device(self, q, qd, qdd, links, local, J=None, vel=None, acc=None, stream=None):
        """Device version of point_motion_host on the SoA layout: q float32 CUDA tensor [n_q, n_stride], qd and qdd [n_qd, n_stride] (or
        None); J [6K * n_qd, n_stride], vel and acc [6K, n_stride] float64 CUDA tensors (any may be None, not all three), entry (point k,
        row r, column c) of J at row (6k + r) * n_qd + c.  The point table is host data.  Asynchronous on the stream."""
        st = _stream(stream)
        keep, K, lp, cp = self._kin_args(links, local)
        self._check(self._L.tds_b200_point_motion_device(self._h, _ptr(q), _ptr(qd), _ptr(qdd), K, lp, cp, _ptr(J), _ptr(vel), _ptr(acc), st),
                    "point_motion_device")

    def point_motion_jvp_host(self, q, qd, links, local, qdd=None, t_q=None, t_qd=None, t_qdd=None):
        """Directional derivatives (dJ [n, K, 6, n_qd, m], dvel [n, K, 6, m], dacc [n, K, 6, m]) of the outputs of point_motion_host along
        m tangents t_q [n, n_q, m], t_qd and t_qdd [n, n_qd, m] (each may be None, not all); tangents given as [n, dim] are m = 1 and
        drop the last axis."""
        q = self._inv_in(q, self.n_q, "q")
        qd, qdd = self._inv_in(qd, self.n_qd, "qd"), self._inv_in(qdd, self.n_qd, "qdd")
        if all(t is None for t in (t_q, t_qd, t_qdd)):
            raise ValueError("at least one tangent is expected")
        ts, m, single = self._tangents([(t_q, self.n_q), (t_qd, self.n_qd), (t_qdd, self.n_qd)])
        keep, K, lp, cp = self._kin_args(links, local)
        n = self.n_envs
        dJ, dvel, dacc = np.zeros((n, K, 6, self.n_qd, m)), np.zeros((n, K, 6, m)), np.zeros((n, K, 6, m))
        self._check(self._L.tds_b200_point_motion_jvp_host(self._h, _dp(q), _dp(qd), _dp(qdd), K, lp, cp, m, *(_dp(t) for t in ts), _dp(dJ),
                                                           _dp(dvel), _dp(dacc)), "point_motion_jvp_host")
        return (dJ[..., 0], dvel[..., 0], dacc[..., 0]) if single else (dJ, dvel, dacc)

    def point_motion_jvp_device(self, q, qd, qdd, links, local, m, t_q, t_qd, t_qdd, t_J=None, t_vel=None, t_acc=None, stream=None):
        """Device version of point_motion_jvp_host: q float32 [n_q, n_stride], qd and qdd [n_qd, n_stride] (or None); t_q [n_q * m,
        n_stride], t_qd and t_qdd [n_qd * m, n_stride] (each may be None, not all), t_J [6K * n_qd * m, n_stride], t_vel and t_acc [6K * m,
        n_stride] (any may be None, not all three) float64 CUDA tensors, entry (r, j) at row r * m + j.  Asynchronous on the stream."""
        st = _stream(stream)
        keep, K, lp, cp = self._kin_args(links, local)
        self._check(self._L.tds_b200_point_motion_jvp_device(self._h, _ptr(q), _ptr(qd), _ptr(qdd), K, lp, cp, int(m), _ptr(t_q), _ptr(t_qd),
                                                             _ptr(t_qdd), _ptr(t_J), _ptr(t_vel), _ptr(t_acc), st), "point_motion_jvp_device")

    def point_motion_vjp_host(self, q, qd, links, local, qdd=None, G_J=None, G_vel=None, G_acc=None):
        """Cotangents G_J [n, K, 6, n_qd], G_vel and G_acc [n, K, 6] (None: zero, not all three) -> (g_q [n, n_q], g_qd [n, n_qd], g_qdd
        [n, n_qd]) = sum G * d(outputs)/dx."""
        q = self._inv_in(q, self.n_q, "q")
        qd, qdd = self._inv_in(qd, self.n_qd, "qd"), self._inv_in(qdd, self.n_qd, "qdd")
        keep, K, lp, cp = self._kin_args(links, local)
        if G_J is None and G_vel is None and G_acc is None:
            raise ValueError("at least one cotangent is expected")
        n = self.n_envs
        G_J = None if G_J is None else self._inv_in(np.reshape(G_J, (n, -1)), 6 * K * self.n_qd, "G_J")
        G_vel = None if G_vel is None else self._inv_in(np.reshape(G_vel, (n, -1)), 6 * K, "G_vel")
        G_acc = None if G_acc is None else self._inv_in(np.reshape(G_acc, (n, -1)), 6 * K, "G_acc")
        g_q, g_qd, g_qdd = np.zeros((n, self.n_q)), np.zeros((n, self.n_qd)), np.zeros((n, self.n_qd))
        self._check(self._L.tds_b200_point_motion_vjp_host(self._h, _dp(q), _dp(qd), _dp(qdd), K, lp, cp, _dp(G_J), _dp(G_vel), _dp(G_acc),
                                                           _dp(g_q), _dp(g_qd), _dp(g_qdd)), "point_motion_vjp_host")
        return g_q, g_qd, g_qdd

    def point_motion_vjp_device(self, q, qd, qdd, links, local, G_J, G_vel, G_acc, g_q, g_qd, g_qdd, stream=None):
        """Device version of point_motion_vjp_host: q float32 [n_q, n_stride], qd and qdd [n_qd, n_stride] (or None), cotangents float64
        in the layouts of point_motion_device (None: zero, not all three), g_q [n_q, n_stride], g_qd and g_qdd [n_qd, n_stride] float64
        CUDA tensors (each may be None, not all).  Asynchronous on the stream."""
        st = _stream(stream)
        keep, K, lp, cp = self._kin_args(links, local)
        self._check(self._L.tds_b200_point_motion_vjp_device(self._h, _ptr(q), _ptr(qd), _ptr(qdd), K, lp, cp, _ptr(G_J), _ptr(G_vel),
                                                             _ptr(G_acc), _ptr(g_q), _ptr(g_qd), _ptr(g_qdd), st), "point_motion_vjp_device")

    # ---- joint-torque and energy regressors of the inertial parameters (DESIGN.md section 7.19) ----
    @property
    def n_pi(self):
        """Columns of the regressors: the physical-parameter ids from 2 on (tds_b200.model.regressor_names)."""
        return 12 * self.n_links + 10

    def regressor_host(self, q, qd=None, qdd=None):
        """(Y [n, n_qd, n_pi], yT [n, n_pi], yV [n, n_pi]) float64 at the fp32-rounded q [n, n_q], qd and qdd [n, n_qd] (None: zero):
        inverse_dynamics_host(q, qd, qdd) = Y @ pi, the kinetic energy 1/2 qd^T M qd = yT . pi and the potential energy yV . pi, for the
        barycentric inertial parameters, stiffness and damping pi of tds_b200.model.inertial_parameters.  Installed physical parameters
        do not enter."""
        q = self._inv_in(q, self.n_q, "q")
        qd, qdd = self._inv_in(qd, self.n_qd, "qd"), self._inv_in(qdd, self.n_qd, "qdd")
        n = self.n_envs
        Y, yT, yV = np.zeros((n, self.n_qd, self.n_pi)), np.zeros((n, self.n_pi)), np.zeros((n, self.n_pi))
        self._check(self._L.tds_b200_regressor_host(self._h, _dp(q), _dp(qd), _dp(qdd), _dp(Y), _dp(yT), _dp(yV)), "regressor_host")
        return Y, yT, yV

    def regressor_device(self, q, qd, qdd, Y=None, yT=None, yV=None, stream=None):
        """Device version of regressor_host on the SoA layout: q float32 CUDA tensor [n_q, n_stride], qd and qdd [n_qd, n_stride] (or
        None); Y [n_qd * n_pi, n_stride] (entry (r, c) at row r * n_pi + c), yT and yV [n_pi, n_stride] float64 CUDA tensors (any may be
        None, not all three).  Asynchronous on the stream."""
        st = _stream(stream)
        self._check(self._L.tds_b200_regressor_device(self._h, _ptr(q), _ptr(qd), _ptr(qdd), _ptr(Y), _ptr(yT), _ptr(yV), st),
                    "regressor_device")

    def regressor_jvp_host(self, q, qd=None, qdd=None, t_q=None, t_qd=None, t_qdd=None):
        """Directional derivatives (dY [n, n_qd, n_pi, m], dyT [n, n_pi, m], dyV [n, n_pi, m]) of the outputs of regressor_host along m
        tangents t_q [n, n_q, m], t_qd and t_qdd [n, n_qd, m] (each may be None, not all); tangents given as [n, dim] are m = 1 and drop
        the last axis."""
        q = self._inv_in(q, self.n_q, "q")
        qd, qdd = self._inv_in(qd, self.n_qd, "qd"), self._inv_in(qdd, self.n_qd, "qdd")
        if all(t is None for t in (t_q, t_qd, t_qdd)):
            raise ValueError("at least one tangent is expected")
        ts, m, single = self._tangents([(t_q, self.n_q), (t_qd, self.n_qd), (t_qdd, self.n_qd)])
        n = self.n_envs
        dY, dyT, dyV = np.zeros((n, self.n_qd, self.n_pi, m)), np.zeros((n, self.n_pi, m)), np.zeros((n, self.n_pi, m))
        self._check(self._L.tds_b200_regressor_jvp_host(self._h, _dp(q), _dp(qd), _dp(qdd), m, *(_dp(t) for t in ts), _dp(dY), _dp(dyT),
                                                        _dp(dyV)), "regressor_jvp_host")
        return (dY[..., 0], dyT[..., 0], dyV[..., 0]) if single else (dY, dyT, dyV)

    def regressor_jvp_device(self, q, qd, qdd, m, t_q, t_qd, t_qdd, t_Y=None, t_yT=None, t_yV=None, stream=None):
        """Device version of regressor_jvp_host: q float32 [n_q, n_stride], qd and qdd [n_qd, n_stride] (or None); t_q [n_q * m,
        n_stride], t_qd and t_qdd [n_qd * m, n_stride] (each may be None, not all), t_Y [n_qd * n_pi * m, n_stride], t_yT and t_yV
        [n_pi * m, n_stride] (any may be None, not all three) float64 CUDA tensors, entry (r, j) at row r * m + j.  Asynchronous."""
        st = _stream(stream)
        self._check(self._L.tds_b200_regressor_jvp_device(self._h, _ptr(q), _ptr(qd), _ptr(qdd), int(m), _ptr(t_q), _ptr(t_qd), _ptr(t_qdd),
                                                          _ptr(t_Y), _ptr(t_yT), _ptr(t_yV), st), "regressor_jvp_device")

    def regressor_vjp_host(self, q, qd=None, qdd=None, G_Y=None, G_yT=None, G_yV=None):
        """Cotangents G_Y [n, n_qd, n_pi], G_yT and G_yV [n, n_pi] (None: zero, not all three) -> (g_q [n, n_q], g_qd [n, n_qd], g_qdd
        [n, n_qd]) = sum G * d(outputs)/dx."""
        q = self._inv_in(q, self.n_q, "q")
        qd, qdd = self._inv_in(qd, self.n_qd, "qd"), self._inv_in(qdd, self.n_qd, "qdd")
        if G_Y is None and G_yT is None and G_yV is None:
            raise ValueError("at least one cotangent is expected")
        n = self.n_envs
        G_Y = None if G_Y is None else self._inv_in(np.reshape(G_Y, (n, -1)), self.n_qd * self.n_pi, "G_Y")
        G_yT = None if G_yT is None else self._inv_in(G_yT, self.n_pi, "G_yT")
        G_yV = None if G_yV is None else self._inv_in(G_yV, self.n_pi, "G_yV")
        g_q, g_qd, g_qdd = np.zeros((n, self.n_q)), np.zeros((n, self.n_qd)), np.zeros((n, self.n_qd))
        self._check(self._L.tds_b200_regressor_vjp_host(self._h, _dp(q), _dp(qd), _dp(qdd), _dp(G_Y), _dp(G_yT), _dp(G_yV), _dp(g_q),
                                                        _dp(g_qd), _dp(g_qdd)), "regressor_vjp_host")
        return g_q, g_qd, g_qdd

    def regressor_vjp_device(self, q, qd, qdd, G_Y, G_yT, G_yV, g_q, g_qd, g_qdd, stream=None):
        """Device version of regressor_vjp_host: q float32 [n_q, n_stride], qd and qdd [n_qd, n_stride] (or None), cotangents float64 in
        the layouts of regressor_device (None: zero, not all three), g_q [n_q, n_stride], g_qd and g_qdd [n_qd, n_stride] float64 CUDA
        tensors (each may be None, not all).  Asynchronous on the stream."""
        st = _stream(stream)
        self._check(self._L.tds_b200_regressor_vjp_device(self._h, _ptr(q), _ptr(qd), _ptr(qdd), _ptr(G_Y), _ptr(G_yT), _ptr(G_yV),
                                                          _ptr(g_q), _ptr(g_qd), _ptr(g_qdd), st), "regressor_vjp_device")

    # ---- inverse mass matrix and operational-space inverse inertia (DESIGN.md section 7.20) ----
    def _minv_points(self, links, local):
        """The point table of the mass_inverse methods (None: no points, K = 0)."""
        return self._kin_args([] if links is None else links, np.zeros((0, 3)) if local is None else local)

    def mass_inverse_host(self, q, links=None, local=None):
        """(Minv [n, n_qd, n_qd], Linv [n, 6K, 6K] or None without points) float64 at the fp32-rounded q [n, n_q]: the inverse of
        mass_matrix_host(q) (bitwise symmetric; for a floating base not the forward dynamics' dqdd/dtau), and the operational-space
        inverse inertia J Minv J^T of the point table links [K] / local [K, 3] (K <= 16), J the spatial point Jacobian of
        point_motion_host ([n, K, 6, n_qd] flattened to 6K rows).  Installed masses, centres of mass and inertias enter."""
        q = self._inv_in(q, self.n_q, "q")
        keep, K, lp, cp = self._minv_points(links, local)
        n = self.n_envs
        Minv, Linv = np.zeros((n, self.n_qd, self.n_qd)), (np.zeros((n, 6 * K, 6 * K)) if K else None)
        self._check(self._L.tds_b200_mass_inverse_host(self._h, _dp(q), K, lp, cp, _dp(Minv), _dp(Linv)), "mass_inverse_host")
        return Minv, Linv

    def mass_inverse_device(self, q, links, local, Minv=None, Linv=None, stream=None):
        """Device version of mass_inverse_host on the SoA layout: q float32 CUDA tensor [n_q, n_stride]; Minv [n_qd * n_qd, n_stride] and
        Linv [36 K^2, n_stride] float64 CUDA tensors (either may be None, not both), entry (r, c) at row r * n_qd + c (r * 6K + c).  The
        point table (None: none) is host data.  Asynchronous on the stream."""
        st = _stream(stream)
        keep, K, lp, cp = self._minv_points(links, local)
        self._check(self._L.tds_b200_mass_inverse_device(self._h, _ptr(q), K, lp, cp, _ptr(Minv), _ptr(Linv), st), "mass_inverse_device")

    def mass_inverse_jvp_host(self, q, links=None, local=None, t_q=None, t_par=None):
        """Directional derivatives of the outputs of mass_inverse_host along m tangents t_q [n, n_q, m] of q and t_par [n, k, m] of the
        installed parameters (either may be None, not both): (Minv, Linv, dMinv [n, n_qd, n_qd, m], dLinv [n, 6K, 6K, m] or None);
        tangents given as [n, dim] are m = 1 and drop the last axis."""
        q = self._inv_in(q, self.n_q, "q")
        keep, K, lp, cp = self._minv_points(links, local)
        (tq, tp), m, single = self._tangents([(t_q, self.n_q), (t_par, len(self.param_ids))], names="t_q and t_par")
        n, nd = self.n_envs, self.n_qd
        Minv, dMinv = np.zeros((n, nd, nd)), np.zeros((n, nd, nd, max(m, 1)))
        Linv, dLinv = (np.zeros((n, 6 * K, 6 * K)), np.zeros((n, 6 * K, 6 * K, max(m, 1)))) if K else (None, None)
        self._check(self._L.tds_b200_mass_inverse_jvp_host(self._h, _dp(q), K, lp, cp, m, _dp(tq), _dp(tp), _dp(Minv), _dp(Linv), _dp(dMinv),
                                                           _dp(dLinv)), "mass_inverse_jvp_host")
        if single:
            dMinv, dLinv = dMinv[..., 0], (None if dLinv is None else dLinv[..., 0])
        return Minv, Linv, dMinv, dLinv

    def mass_inverse_jvp_device(self, q, links, local, m, t_q, t_par, t_Minv=None, t_Linv=None, Minv=None, Linv=None, stream=None):
        """Device version of mass_inverse_jvp_host: q float32 [n_q, n_stride]; t_q [n_q * m, n_stride], t_par [k * m, n_stride] (either may
        be None, not both); t_Minv [n_qd^2 * m, n_stride], t_Linv [36 K^2 * m, n_stride] (either may be None, not both), Minv and Linv
        (values, or None) float64 CUDA tensors, entry (r, j) at row r * m + j.  Asynchronous on the stream."""
        st = _stream(stream)
        keep, K, lp, cp = self._minv_points(links, local)
        self._check(self._L.tds_b200_mass_inverse_jvp_device(self._h, _ptr(q), K, lp, cp, int(m), _ptr(t_q), _ptr(t_par), _ptr(Minv),
                                                             _ptr(Linv), _ptr(t_Minv), _ptr(t_Linv), st), "mass_inverse_jvp_device")

    def mass_inverse_vjp_host(self, q, links=None, local=None, G_Minv=None, G_Linv=None):
        """Cotangents G_Minv [n, n_qd, n_qd] and G_Linv [n, 6K, 6K] (None: zero, not both) -> (g_q [n, n_q], g_par [n, k] or None without
        installed parameters) = sum G * d(outputs)/dx."""
        q = self._inv_in(q, self.n_q, "q")
        keep, K, lp, cp = self._minv_points(links, local)
        if G_Minv is None and G_Linv is None:
            raise ValueError("at least one cotangent is expected")
        n = self.n_envs
        G_Minv = None if G_Minv is None else self._inv_in(np.reshape(G_Minv, (n, -1)), self.n_qd * self.n_qd, "G_Minv")
        G_Linv = None if G_Linv is None else self._inv_in(np.reshape(G_Linv, (n, -1)), 36 * K * K, "G_Linv")
        k = len(self.param_ids)
        g_q = np.zeros((n, self.n_q))
        g_par = np.zeros((n, k)) if k else None
        self._check(self._L.tds_b200_mass_inverse_vjp_host(self._h, _dp(q), K, lp, cp, _dp(G_Minv), _dp(G_Linv), _dp(g_q), _dp(g_par)),
                    "mass_inverse_vjp_host")
        return g_q, g_par

    def mass_inverse_vjp_device(self, q, links, local, G_Minv, G_Linv, g_q, g_par=None, stream=None):
        """Device version of mass_inverse_vjp_host: q float32 [n_q, n_stride], cotangents float64 in the layouts of mass_inverse_device
        (None: zero, not both), g_q [n_q, n_stride] and g_par [k, n_stride] float64 CUDA tensors (either may be None, not both).
        Asynchronous on the stream."""
        st = _stream(stream)
        keep, K, lp, cp = self._minv_points(links, local)
        self._check(self._L.tds_b200_mass_inverse_vjp_device(self._h, _ptr(q), K, lp, cp, _ptr(G_Minv), _ptr(G_Linv), _ptr(g_q), _ptr(g_par),
                                                             st), "mass_inverse_vjp_device")

    # ---- Coriolis matrix C(q, qd) (DESIGN.md section 7.22) ----
    def coriolis_host(self, q, qd=None):
        """C [n, n_qd, n_qd] float64 at the fp32-rounded q [n, n_q] and qd [n, n_qd] (None: zero, C = 0), in the coordinates of
        mass_matrix_host: Echeandia & Wensing's factorisation, so that C qd is the velocity part of the bias forces (inverse_dynamics_host(q,
        qd) - inverse_dynamics_host(q) without joint damping) and C + C^T is the time derivative of M along qd.  Installed masses, centres
        of mass and inertias apply per environment; stiffness, damping, friction and restitution do not enter (include/tds_b200.h)."""
        q = self._inv_in(q, self.n_q, "q")
        qd = self._inv_in(qd, self.n_qd, "qd")
        C = np.zeros((self.n_envs, self.n_qd, self.n_qd))
        self._check(self._L.tds_b200_coriolis_host(self._h, _dp(q), _dp(qd), _dp(C)), "coriolis_host")
        return C

    def coriolis_device(self, q, qd, C, stream=None):
        """Device version of coriolis_host on the SoA layout: q float32 CUDA tensor [n_q, n_stride], qd [n_qd, n_stride] (or None), C
        float64 [n_qd * n_qd, n_stride], entry (r, c) at row r * n_qd + c.  Asynchronous on the stream."""
        st = _stream(stream)
        self._check(self._L.tds_b200_coriolis_device(self._h, _ptr(q), _ptr(qd), _ptr(C), st), "coriolis_device")

    def coriolis_jvp_host(self, q, qd=None, t_q=None, t_qd=None, t_par=None):
        """Directional derivatives of C along m tangents t_q [n, n_q, m], t_qd [n, n_qd, m] and t_par [n, k, m] of the installed
        parameters (each may be None, not all): (C, dC [n, n_qd, n_qd, m]); tangents given as [n, dim] are m = 1 and drop the last axis."""
        q = self._inv_in(q, self.n_q, "q")
        qd = self._inv_in(qd, self.n_qd, "qd")
        if all(t is None for t in (t_q, t_qd, t_par)):
            raise ValueError("at least one tangent is expected")
        (tq, tqd, tp), m, single = self._tangents([(t_q, self.n_q), (t_qd, self.n_qd), (t_par, len(self.param_ids))])
        n, nd = self.n_envs, self.n_qd
        C, dC = np.zeros((n, nd, nd)), np.zeros((n, nd, nd, m))
        self._check(self._L.tds_b200_coriolis_jvp_host(self._h, _dp(q), _dp(qd), m, _dp(tq), _dp(tqd), _dp(tp), _dp(C), _dp(dC)),
                    "coriolis_jvp_host")
        return C, (dC[..., 0] if single else dC)

    def coriolis_jvp_device(self, q, qd, m, t_q, t_qd, t_par, t_C, C=None, stream=None):
        """Device version of coriolis_jvp_host: q float32 [n_q, n_stride], qd [n_qd, n_stride] (or None); t_q [n_q * m, n_stride], t_qd
        [n_qd * m, n_stride], t_par [k * m, n_stride] (each may be None, not all), t_C [n_qd^2 * m, n_stride] and C [n_qd^2, n_stride] (or
        None) float64 CUDA tensors, entry (r, j) at row r * m + j.  Asynchronous on the stream."""
        st = _stream(stream)
        self._check(self._L.tds_b200_coriolis_jvp_device(self._h, _ptr(q), _ptr(qd), int(m), _ptr(t_q), _ptr(t_qd), _ptr(t_par), _ptr(C),
                                                         _ptr(t_C), st), "coriolis_jvp_device")

    def coriolis_vjp_host(self, q, qd, G):
        """Cotangent G [n, n_qd, n_qd] of C -> (g_q [n, n_q], g_qd [n, n_qd], g_par [n, k] or None without installed parameters)."""
        q = self._inv_in(q, self.n_q, "q")
        qd = self._inv_in(qd, self.n_qd, "qd")
        n = self.n_envs
        G = self._inv_in(np.reshape(G, (n, -1)), self.n_qd * self.n_qd, "G")
        k = len(self.param_ids)
        g_q, g_qd = np.zeros((n, self.n_q)), np.zeros((n, self.n_qd))
        g_par = np.zeros((n, k)) if k else None
        self._check(self._L.tds_b200_coriolis_vjp_host(self._h, _dp(q), _dp(qd), _dp(G), _dp(g_q), _dp(g_qd), _dp(g_par)), "coriolis_vjp_host")
        return g_q, g_qd, g_par

    def coriolis_vjp_device(self, q, qd, G, g_q, g_qd=None, g_par=None, stream=None):
        """Device version of coriolis_vjp_host: q float32 [n_q, n_stride], qd [n_qd, n_stride] (or None), G float64 [n_qd * n_qd, n_stride]
        in C's layout, g_q [n_q, n_stride], g_qd [n_qd, n_stride], g_par [k, n_stride] float64 CUDA tensors (each may be None, not all).
        Asynchronous on the stream."""
        st = _stream(stream)
        self._check(self._L.tds_b200_coriolis_vjp_device(self._h, _ptr(q), _ptr(qd), _ptr(G), _ptr(g_q), _ptr(g_qd), _ptr(g_par), st),
                    "coriolis_vjp_device")

    # ---- point-constrained forward dynamics (DESIGN.md section 7.21) ----
    def _cd_points(self, links, local, dims, damping):
        """The point table (None: no points, K = 0), dims and damping of the constrained_dynamics methods."""
        keep, K, lp, cp = self._minv_points(links, local)
        return keep, K, lp, cp, int(dims), float(damping)

    def constrained_dynamics_host(self, q, qd=None, tau=None, links=None, local=None, dims=3, damping=0.0):
        """(qdd [n, n_qd], f [n, K, dims] or None without points) float64 at the fp32-rounded q [n, n_q], qd and tau [n, n_qd] (None: zero):
        the forward dynamics with the points of links [K] / local [K, 3] (K <= 16) held in their 3 linear rows (dims 3) or all 6 rows
        (dims 6), M qdd - J_c^T f = tau - h and J_c qdd = -d_c - damping f, with M, h and J, d of mass_matrix_host,
        inverse_dynamics_host(q, qd) and point_motion_host(q, qd).  f: the force (dims 3) or wrench [n; f] (dims 6) the constraint applies
        at each point, world axes.  K = 0: qdd = M^-1 (tau - h).  Installed masses, centres of mass, inertias, stiffness and damping
        enter.  An environment whose constraint system is not positive definite gets NaN outputs."""
        q = self._inv_in(q, self.n_q, "q")
        qd, tau = self._inv_in(qd, self.n_qd, "qd"), self._inv_in(tau, self.n_qd, "tau")
        keep, K, lp, cp, dims, eps = self._cd_points(links, local, dims, damping)
        n = self.n_envs
        qdd, f = np.zeros((n, self.n_qd)), (np.zeros((n, K, dims)) if K else None)
        self._check(self._L.tds_b200_constrained_dynamics_host(self._h, _dp(q), _dp(qd), _dp(tau), K, lp, cp, dims, eps, _dp(qdd), _dp(f)),
                    "constrained_dynamics_host")
        return qdd, f

    def constrained_dynamics_device(self, q, qd, tau, links, local, dims, damping, qdd=None, f=None, stream=None):
        """Device version of constrained_dynamics_host on the SoA layout: q float32 CUDA tensor [n_q, n_stride], qd and tau [n_qd, n_stride]
        (or None); qdd [n_qd, n_stride] and f [dims K, n_stride] float64 CUDA tensors (either may be None, not both), component r of point
        k at row dims k + r.  The point table (None: none) is host data.  Asynchronous on the stream."""
        st = _stream(stream)
        keep, K, lp, cp, dims, eps = self._cd_points(links, local, dims, damping)
        self._check(self._L.tds_b200_constrained_dynamics_device(self._h, _ptr(q), _ptr(qd), _ptr(tau), K, lp, cp, dims, eps, _ptr(qdd),
                                                                 _ptr(f), st), "constrained_dynamics_device")

    def constrained_dynamics_jvp_host(self, q, qd=None, tau=None, links=None, local=None, dims=3, damping=0.0, t_q=None, t_qd=None,
                                      t_tau=None, t_par=None):
        """Directional derivatives of the outputs of constrained_dynamics_host along m tangents t_q [n, n_q, m], t_qd and t_tau [n, n_qd, m]
        and t_par [n, k, m] of the installed parameters (each may be None, not all): (qdd, f, dqdd [n, n_qd, m], df [n, K, dims, m] or
        None); tangents given as [n, dim] are m = 1 and drop the last axis."""
        q = self._inv_in(q, self.n_q, "q")
        qd, tau = self._inv_in(qd, self.n_qd, "qd"), self._inv_in(tau, self.n_qd, "tau")
        keep, K, lp, cp, dims, eps = self._cd_points(links, local, dims, damping)
        ts, m, single = self._tangents([(t_q, self.n_q), (t_qd, self.n_qd), (t_tau, self.n_qd), (t_par, len(self.param_ids))])
        n, nd = self.n_envs, self.n_qd
        qdd, dqdd = np.zeros((n, nd)), np.zeros((n, nd, max(m, 1)))
        f, df = (np.zeros((n, K, dims)), np.zeros((n, K, dims, max(m, 1)))) if K else (None, None)
        self._check(self._L.tds_b200_constrained_dynamics_jvp_host(self._h, _dp(q), _dp(qd), _dp(tau), K, lp, cp, dims, eps, m,
                                                                   *(_dp(t) for t in ts), _dp(qdd), _dp(f), _dp(dqdd), _dp(df)),
                    "constrained_dynamics_jvp_host")
        if single:
            dqdd, df = dqdd[..., 0], (None if df is None else df[..., 0])
        return qdd, f, dqdd, df

    def constrained_dynamics_jvp_device(self, q, qd, tau, links, local, dims, damping, m, t_q, t_qd, t_tau, t_par, t_qdd=None, t_f=None,
                                        qdd=None, f=None, stream=None):
        """Device version of constrained_dynamics_jvp_host: q float32 [n_q, n_stride], qd and tau [n_qd, n_stride] (or None); t_q [n_q * m,
        n_stride], t_qd and t_tau [n_qd * m, n_stride], t_par [k * m, n_stride] (each may be None, not all); t_qdd [n_qd * m, n_stride],
        t_f [dims K m, n_stride] (either may be None, not both), qdd and f (values, or None) float64 CUDA tensors, entry (r, j) at row
        r * m + j.  Asynchronous on the stream."""
        st = _stream(stream)
        keep, K, lp, cp, dims, eps = self._cd_points(links, local, dims, damping)
        self._check(self._L.tds_b200_constrained_dynamics_jvp_device(self._h, _ptr(q), _ptr(qd), _ptr(tau), K, lp, cp, dims, eps, int(m),
                                                                     _ptr(t_q), _ptr(t_qd), _ptr(t_tau), _ptr(t_par), _ptr(qdd), _ptr(f),
                                                                     _ptr(t_qdd), _ptr(t_f), st), "constrained_dynamics_jvp_device")

    def constrained_dynamics_vjp_host(self, q, qd=None, tau=None, links=None, local=None, dims=3, damping=0.0, G_qdd=None, G_f=None):
        """Cotangents G_qdd [n, n_qd] and G_f [n, K, dims] (None: zero, not both) -> (g_q [n, n_q], g_qd [n, n_qd], g_tau [n, n_qd], g_par
        [n, k] or None without installed parameters) = sum G * d(outputs)/dx."""
        q = self._inv_in(q, self.n_q, "q")
        qd, tau = self._inv_in(qd, self.n_qd, "qd"), self._inv_in(tau, self.n_qd, "tau")
        keep, K, lp, cp, dims, eps = self._cd_points(links, local, dims, damping)
        if G_qdd is None and G_f is None:
            raise ValueError("at least one cotangent is expected")
        n, nd, k = self.n_envs, self.n_qd, len(self.param_ids)
        G_qdd = None if G_qdd is None else self._inv_in(G_qdd, nd, "G_qdd")
        G_f = None if G_f is None else self._inv_in(np.reshape(G_f, (n, -1)), dims * K, "G_f")
        g_q, g_qd, g_tau = np.zeros((n, self.n_q)), np.zeros((n, nd)), np.zeros((n, nd))
        g_par = np.zeros((n, k)) if k else None
        self._check(self._L.tds_b200_constrained_dynamics_vjp_host(self._h, _dp(q), _dp(qd), _dp(tau), K, lp, cp, dims, eps, _dp(G_qdd),
                                                                   _dp(G_f), _dp(g_q), _dp(g_qd), _dp(g_tau), _dp(g_par)),
                    "constrained_dynamics_vjp_host")
        return g_q, g_qd, g_tau, g_par

    def constrained_dynamics_vjp_device(self, q, qd, tau, links, local, dims, damping, G_qdd, G_f, g_q, g_qd, g_tau, g_par=None,
                                        stream=None):
        """Device version of constrained_dynamics_vjp_host: q float32 [n_q, n_stride], qd and tau [n_qd, n_stride] (or None), cotangents
        float64 in the layouts of constrained_dynamics_device (None: zero, not both), g_q [n_q, n_stride], g_qd and g_tau [n_qd, n_stride],
        g_par [k, n_stride] float64 CUDA tensors (each may be None, not all).  Asynchronous on the stream."""
        st = _stream(stream)
        keep, K, lp, cp, dims, eps = self._cd_points(links, local, dims, damping)
        self._check(self._L.tds_b200_constrained_dynamics_vjp_device(self._h, _ptr(q), _ptr(qd), _ptr(tau), K, lp, cp, dims, eps, _ptr(G_qdd),
                                                                     _ptr(G_f), _ptr(g_q), _ptr(g_qd), _ptr(g_tau), _ptr(g_par), st),
                    "constrained_dynamics_vjp_device")

    # ---- derivatives of the forward dynamics (DESIGN.md section 7.24) ----
    def forward_dynamics_derivatives_host(self, q, qd=None, tau=None):
        """(qdd [n, n_qd], dqdd_dq, dqdd_dqd, dqdd_dtau [n, n_qd, n_qd]) float64 at the fp32-rounded q [n, n_q], qd and tau [n, n_qd] (None:
        zero): qdd = M^-1 (tau - h) is constrained_dynamics_host's qdd without points, dqdd_dq = -M^-1 dtau_dq and dqdd_dqd = -M^-1
        dtau_dqd with the inverse dynamics' derivatives taken at that qdd in fp64, dqdd_dtau = M^-1 (mass_inverse_host's).  Row r = qdd_r,
        columns in M's coordinates: column k of dqdd_dq is constrained_dynamics_jvp_host along t_q = dq_dt(q, e_k) (include/tds_b200.h)."""
        q = self._inv_in(q, self.n_q, "q")
        qd, tau = self._inv_in(qd, self.n_qd, "qd"), self._inv_in(tau, self.n_qd, "tau")
        n, nd = self.n_envs, self.n_qd
        qdd, a, b, c = np.zeros((n, nd)), np.zeros((n, nd, nd)), np.zeros((n, nd, nd)), np.zeros((n, nd, nd))
        self._check(self._L.tds_b200_forward_dynamics_derivatives_host(self._h, _dp(q), _dp(qd), _dp(tau), _dp(qdd), _dp(a), _dp(b), _dp(c)),
                    "forward_dynamics_derivatives_host")
        return qdd, a, b, c

    def forward_dynamics_derivatives_device(self, q, qd, tau, qdd, dqdd_dq, dqdd_dqd, dqdd_dtau, stream=None):
        """Device version of forward_dynamics_derivatives_host on the SoA layout: q float32 CUDA tensor [n_q, n_stride], qd and tau [n_qd,
        n_stride] (either may be None); qdd [n_qd, n_stride] and the matrices [n_qd * n_qd, n_stride] float64 CUDA tensors (each may be
        None, not all).  Asynchronous on the stream."""
        st = _stream(stream)
        self._check(self._L.tds_b200_forward_dynamics_derivatives_device(self._h, _ptr(q), _ptr(qd), _ptr(tau), _ptr(qdd), _ptr(dqdd_dq),
                                                                         _ptr(dqdd_dqd), _ptr(dqdd_dtau), st),
                    "forward_dynamics_derivatives_device")

    def forward_dynamics_derivatives_jvp_host(self, q, qd=None, tau=None, t_q=None, t_qd=None, t_tau=None, t_par=None):
        """Directional derivatives of the four outputs of forward_dynamics_derivatives_host along m tangents t_q [n, n_q, m], t_qd and t_tau
        [n, n_qd, m] and t_par [n, k, m] (each may be None, not all): (qdd, dqdd_dq, dqdd_dqd, dqdd_dtau, t_qdd [n, n_qd, m], t_dqdd_dq,
        t_dqdd_dqd, t_dqdd_dtau [n, n_qd, n_qd, m]); tangents given as [n, dim] are m = 1 and drop the last axis."""
        q = self._inv_in(q, self.n_q, "q")
        qd, tau = self._inv_in(qd, self.n_qd, "qd"), self._inv_in(tau, self.n_qd, "tau")
        if all(t is None for t in (t_q, t_qd, t_tau, t_par)):
            raise ValueError("at least one tangent is expected")
        ts, m, single = self._tangents([(t_q, self.n_q), (t_qd, self.n_qd), (t_tau, self.n_qd), (t_par, len(self.param_ids))])
        n, nd = self.n_envs, self.n_qd
        vals = [np.zeros((n, nd))] + [np.zeros((n, nd, nd)) for _ in range(3)]
        tans = [np.zeros((n, nd, m))] + [np.zeros((n, nd, nd, m)) for _ in range(3)]
        self._check(self._L.tds_b200_forward_dynamics_derivatives_jvp_host(self._h, _dp(q), _dp(qd), _dp(tau), m, *(_dp(t) for t in ts),
                                                                           *(_dp(x) for x in vals + tans)),
                    "forward_dynamics_derivatives_jvp_host")
        if single:
            tans = [t[..., 0] for t in tans]
        return tuple(vals + tans)

    def forward_dynamics_derivatives_jvp_device(self, q, qd, tau, m, t_q, t_qd, t_tau, t_par, t_qdd, t_dqdd_dq, t_dqdd_dqd, t_dqdd_dtau,
                                                qdd=None, dqdd_dq=None, dqdd_dqd=None, dqdd_dtau=None, stream=None):
        """Device version of forward_dynamics_derivatives_jvp_host: q float32 [n_q, n_stride], qd and tau [n_qd, n_stride] (or None); t_q
        [n_q * m, n_stride], t_qd and t_tau [n_qd * m, n_stride], t_par [k * m, n_stride] (each may be None, not all); t_qdd [n_qd * m,
        n_stride] and the matrices' tangents [n_qd * n_qd * m, n_stride] (each may be None, not all), and the values (or None) float64
        CUDA tensors, entry (r, j) at row r * m + j.  Asynchronous on the stream."""
        st = _stream(stream)
        self._check(self._L.tds_b200_forward_dynamics_derivatives_jvp_device(
            self._h, _ptr(q), _ptr(qd), _ptr(tau), int(m), _ptr(t_q), _ptr(t_qd), _ptr(t_tau), _ptr(t_par), _ptr(qdd), _ptr(dqdd_dq),
            _ptr(dqdd_dqd), _ptr(dqdd_dtau), _ptr(t_qdd), _ptr(t_dqdd_dq), _ptr(t_dqdd_dqd), _ptr(t_dqdd_dtau), st),
            "forward_dynamics_derivatives_jvp_device")

    def forward_dynamics_derivatives_vjp_host(self, q, qd=None, tau=None, G_qdd=None, G_dq=None, G_dqd=None, G_dtau=None):
        """Cotangents G_qdd [n, n_qd], G_dq, G_dqd, G_dtau [n, n_qd, n_qd] of the four outputs (each may be None: zero, not all) -> (g_q [n,
        n_q], g_qd [n, n_qd], g_tau [n, n_qd], g_par [n, k] or None without installed parameters)."""
        q = self._inv_in(q, self.n_q, "q")
        qd, tau = self._inv_in(qd, self.n_qd, "qd"), self._inv_in(tau, self.n_qd, "tau")
        if all(G is None for G in (G_qdd, G_dq, G_dqd, G_dtau)):
            raise ValueError("at least one cotangent is expected")
        n, nd, nn, k = self.n_envs, self.n_qd, self.n_qd * self.n_qd, len(self.param_ids)
        G_qdd = None if G_qdd is None else self._inv_in(G_qdd, nd, "G_qdd")
        G_dq, G_dqd, G_dtau = (None if G is None else self._inv_in(np.reshape(G, (n, nn)), nn, w)
                               for G, w in ((G_dq, "G_dq"), (G_dqd, "G_dqd"), (G_dtau, "G_dtau")))
        g_q, g_qd, g_tau = np.zeros((n, self.n_q)), np.zeros((n, nd)), np.zeros((n, nd))
        g_par = np.zeros((n, k)) if k else None
        self._check(self._L.tds_b200_forward_dynamics_derivatives_vjp_host(self._h, _dp(q), _dp(qd), _dp(tau), _dp(G_qdd), _dp(G_dq), _dp(G_dqd),
                                                                           _dp(G_dtau), _dp(g_q), _dp(g_qd), _dp(g_tau), _dp(g_par)),
                    "forward_dynamics_derivatives_vjp_host")
        return g_q, g_qd, g_tau, g_par

    def forward_dynamics_derivatives_vjp_device(self, q, qd, tau, G_qdd, G_dq, G_dqd, G_dtau, g_q, g_qd, g_tau, g_par=None, stream=None):
        """Device version of forward_dynamics_derivatives_vjp_host: q float32 [n_q, n_stride], qd and tau [n_qd, n_stride] (or None),
        cotangents float64 in the layouts of forward_dynamics_derivatives_device (each may be None, not all), g_q [n_q, n_stride], g_qd and
        g_tau [n_qd, n_stride], g_par [k, n_stride] float64 CUDA tensors (each may be None, not all).  Asynchronous on the stream."""
        st = _stream(stream)
        self._check(self._L.tds_b200_forward_dynamics_derivatives_vjp_device(self._h, _ptr(q), _ptr(qd), _ptr(tau), _ptr(G_qdd), _ptr(G_dq),
                                                                             _ptr(G_dqd), _ptr(G_dtau), _ptr(g_q), _ptr(g_qd), _ptr(g_tau),
                                                                             _ptr(g_par), st),
                    "forward_dynamics_derivatives_vjp_device")

    def jacobian_chunk(self):
        """Directions (Jacobian columns or JVP tangents) one launch of the dual-number step takes; more run in several launches."""
        return self._L.tds_b200_jacobian_chunk(self._h)

    def vjp_tape_info(self):
        """(tape capacity in nodes per lane, environments per chunk) of the reverse-mode path as it stands."""
        info = (ctypes.c_int * 2)()
        self._check(self._L.tds_b200_vjp_tape_info(self._h, info), "vjp_tape_info")
        return info[0], info[1]

    def integrate_host(self, q, qd, qdd, update_q=True):
        """integrate_euler (update_q) / integrate_euler_qdd of one state vector per environment, on the device
        (tds_b200_integrate_euler{,_qdd}_device); host arrays [n_q], [n_qd] for a one-environment simulator or [n, dim]."""
        import torch
        dev = f"cuda:{self.device}"
        def up(a, dim):
            t = torch.zeros((max(dim, 1), self.n_stride), dtype=torch.float32, device=dev)
            a = np.asarray(a, dtype=np.float64).reshape(-1, dim) if dim else np.zeros((self.n_envs, 0))
            if dim:
                t[:dim, :self.n_envs] = torch.tensor(np.ascontiguousarray(a.T), dtype=torch.float32)
            return t
        tq, tqd, tqdd = up(q, self.n_q), up(qd, self.n_qd), up(qdd, self.n_qd)
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        if update_q:
            self._check(self._L.tds_b200_integrate_euler_device(self._h, _ptr(tq), _ptr(tqd), _ptr(tqdd), st), "integrate_euler")
        else:
            self._check(self._L.tds_b200_integrate_euler_qdd_device(self._h, _ptr(tqd), _ptr(tqdd), st), "integrate_euler_qdd")
        torch.cuda.synchronize()
        qo = tq[:self.n_q, :self.n_envs].T.cpu().numpy().astype(np.float64)
        qdo = tqd[:self.n_qd, :self.n_envs].T.cpu().numpy().astype(np.float64)
        single = np.asarray(q).ndim == 1
        return (qo[0], qdo[0]) if single else (qo, qdo)

    def contact_pairs(self):
        """(body_a, link_a, body_b, link_b) of every candidate contact point, reference enumeration order
        (World::compute_contacts_multi_body_internal, src/world.hpp:212-281): what World::mb_contacts_ lists each step."""
        t = np.zeros((max(self.n_contact_points, 1), 4), dtype=np.int32)
        k = self._L.tds_b200_contact_pairs(self._h, ctypes.c_void_p(t.ctypes.data), t.shape[0])
        return t[:k]

    def contact_tuples(self):
        """(mb_a, link_a, geom_a, mb_b, link_b, geom_b) of every candidate contact point (geom: index among the link's collision
        shapes): the loop indices of World::compute_contacts_multi_body_internal at which the point is emitted."""
        t = np.zeros((max(self.n_contact_points, 1), 6), dtype=np.int32)
        k = self._L.tds_b200_contact_tuples(self._h, ctypes.c_void_p(t.ctypes.data), t.shape[0])
        return t[:k]

    # ---- resident environment state ----
    def env_set_state(self, q, qd):
        q = np.ascontiguousarray(q, dtype=np.float64)
        qd = np.ascontiguousarray(qd, dtype=np.float64)
        assert q.shape == (self.n_envs, self.n_q) and qd.shape == (self.n_envs, self.n_qd)
        self._check(self._L.tds_b200_env_set_state_host(self._h, _dp(q), _dp(qd)), "env_set_state")

    def env_get_state(self):
        q = np.zeros((self.n_envs, self.n_q))
        qd = np.zeros((self.n_envs, self.n_qd))
        self._check(self._L.tds_b200_env_get_state_host(self._h, _dp(q), _dp(qd)), "env_get_state")
        return q, qd

    def env_step_host(self, actions, obs, rewards, dones):
        """actions/obs/rewards/dones: float32 host arrays (numpy or pinned torch tensors)."""
        def hp(a):
            if a is None:
                return None
            return ctypes.c_void_p(a.data_ptr() if hasattr(a, "data_ptr") else a.ctypes.data)
        self._check(self._L.tds_b200_env_step_host(self._h, hp(actions), hp(obs), hp(rewards), hp(dones)),
                    "env_step_host")

    def num_visuals(self):
        return self._L.tds_b200_num_visuals(self._h)

    def env_step_visual_device(self, actions, positions, orientations, reward=None, done=None, stream=None):
        """Env step that also streams the visual transforms in the instancing renderer's layout:
        positions / orientations are float32 CUDA tensors [n_envs * n_visuals, 4] (xyz1 / quaternion xyzw)."""
        st = _stream(stream)
        self._check(self._L.tds_b200_env_step_visual_device(self._h, _ptr(actions), _ptr(reward), _ptr(done), _ptr(positions),
                                                            _ptr(orientations), st), "env_step_visual_device")

    # ---- environment layer on the device (reset with noise + settle steps, policy rollouts) ----
    def env_reset_device(self, mask=None, noise=None, noise_amp=0.05, seed=0, settle_steps=10, stream=None):
        """mask: float32 CUDA tensor [n] (None = all); noise: float32 CUDA tensor [n_act][n_stride] (None = generated).
        stream None = the simulator's own stream (the one the host-buffer calls use)."""
        st = ctypes.c_void_p(stream.cuda_stream) if stream is not None else None
        self._check(self._L.tds_b200_env_reset_device(self._h, _ptr(mask), _ptr(noise), float(noise_amp), int(seed),
                                                      int(settle_steps), st), "env_reset_device")

    def env_rollout_device(self, policy, rollout_length, shift, total_rewards, steps, stream=None):
        """policy: float32 CUDA tensor [n_params][n_stride]; total_rewards float32 [n], steps int32 [n] CUDA tensors.
        stream None = the simulator's own stream."""
        st = ctypes.c_void_p(stream.cuda_stream) if stream is not None else None
        self._check(self._L.tds_b200_env_rollout_device(self._h, _ptr(policy), int(policy.shape[0]), int(rollout_length),
                                                        float(shift), _ptr(total_rewards), _ptr(steps), st), "env_rollout_device")

    def ars_train_step(self, w, deltas, rollout_length, delta_std=0.025, step_size=0.02, shift=0.0, seed=0, settle_steps=10,
                       obs_stats=None):
        """One ARS iteration without leaving the GPU (ARSLearner::train_step, examples/ars/ars_learner.h:162-190): for the
        directions deltas [n_params][n_stride] (one per environment) a positive and a negative rollout of the linear policy
        w +- delta_std * delta from the same reset (noise keyed by `seed`), then w += step_size * g_hat.  w: float32 CUDA
        tensor [n_params], updated in place.  Returns (r_pos, r_neg) CUDA tensors."""
        import torch
        dev = w.device
        n_params = int(w.numel())
        # everything runs on the simulator's own stream (a NULL stream argument of the env-layer calls means exactly that
        # stream, which is non-blocking: work on torch's default stream would not be ordered against it)
        torch.cuda.current_stream().synchronize()          # w, deltas, obs_stats were produced on the caller's stream
        own = torch.cuda.ExternalStream(self._L.tds_b200_stream(self._h), device=dev)
        sp = ctypes.c_void_p(own.cuda_stream)
        with torch.cuda.stream(own):
            params = torch.empty((n_params, self.n_stride), dtype=torch.float32, device=dev)
            r = [torch.zeros(self.n_stride, dtype=torch.float32, device=dev) for _ in range(2)]
            steps = torch.zeros(self.n_stride, dtype=torch.int32, device=dev)
        self._check(self._L.tds_b200_env_set_obs_stats(self._h, _ptr(obs_stats)), "env_set_obs_stats")
        for k, sign in enumerate((1.0, -1.0)):
            self._check(self._L.tds_b200_ars_perturb_device(self._h, _ptr(w), _ptr(deltas), sign * delta_std, _ptr(params), n_params, sp),
                        "ars_perturb")
            self.env_reset_device(seed=seed, settle_steps=settle_steps, stream=own)
            self.env_rollout_device(params, rollout_length, shift, r[k], steps, stream=own)
        self._check(self._L.tds_b200_ars_update_device(self._h, _ptr(w), _ptr(deltas), _ptr(r[0]), _ptr(r[1]), delta_std, step_size,
                                                       n_params, sp), "ars_update")
        self._check(self._L.tds_b200_env_set_obs_stats(self._h, None), "env_set_obs_stats")
        own.synchronize()
        return r[0], r[1]

    def env_rollout_host(self, policy, rollout_length, shift=0.0, noise=None, noise_amp=0.05, seed=0, settle_steps=10):
        """Reset (noise [n][n_act] or generated) + rollout of per-environment linear policies [n][n_params] (host arrays).
        Returns (total_rewards float64 [n], steps int32 [n])."""
        pol = np.ascontiguousarray(policy, dtype=np.float64)
        assert pol.shape[0] == self.n_envs
        nz = None if noise is None else np.ascontiguousarray(noise, dtype=np.float64)
        tot = np.zeros(self.n_envs)
        steps = np.zeros(self.n_envs, dtype=np.int32)
        self._check(self._L.tds_b200_env_rollout_host(self._h, _dp(pol), int(pol.shape[1]), int(rollout_length), float(shift), _dp(nz),
                                                      float(noise_amp), int(seed), int(settle_steps), _dp(tot),
                                                      ctypes.c_void_p(steps.ctypes.data)), "env_rollout_host")
        return tot, steps

    def bind_env_step_host(self, actions, obs, rewards, dones):
        """Bind the four host buffers once and return a zero-argument callable that performs the env step on them (the
        per-call pointer marshalling of env_step_host is a measurable part of a 40 us step)."""
        def hp(a):
            return None if a is None else ctypes.c_void_p(a.data_ptr() if hasattr(a, "data_ptr") else a.ctypes.data)
        fn, h, args = self._L.tds_b200_env_step_host, self._h, (hp(actions), hp(obs), hp(rewards), hp(dones))
        keep = (actions, obs, rewards, dones)   # the buffers must outlive the callable

        def step():
            rc = fn(h, *args)
            if rc:
                self._check(rc, "env_step_host")
            return keep[1]
        return step

    def env_step_device(self, actions, reward=None, done=None, stream=None):
        st = _stream(stream)
        self._check(self._L.tds_b200_env_step_device(self._h, _ptr(actions), _ptr(reward), _ptr(done), st),
                    "env_step_device")
