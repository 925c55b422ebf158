"""Flat model handling (layout: include/tds_b200_model.h): URDF compile, load / save fixtures."""
import ctypes
import json
import os

import numpy as np

from . import _lib

MAGIC = 20250200
HEADER, BASE, LINK, GEOM, VIS = 16, 13, 34, 18, 13


def compile_urdf(urdf, plane_urdf=None, floating=False):
    """URDF file path or XML text -> flat model (np.float64 array).

    Mirrors UrdfCache::construct (src/urdf/urdf_cache.hpp:74-84) of the reference; `plane_urdf`
    adds the static ground plane body the locomotion environments create first.
    """
    L = _lib.lib()
    u = urdf.encode()
    p = (plane_urdf or "").encode()
    n = L.tds_b200_urdf_to_model(u, p, int(floating), None, 0)
    if n <= 0:
        raise ValueError("URDF compile failed: " + _lib.last_error())
    out = np.zeros(n, dtype=np.float64)
    n2 = L.tds_b200_urdf_to_model(u, p, int(floating), out.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), n)
    if n2 != n:
        raise ValueError("URDF compile failed: " + _lib.last_error())
    return out


def model_dims(model):
    m = np.asarray(model)
    if int(m[0]) != MAGIC:
        raise ValueError("not a tds_b200 flat model")
    return dict(n_links=int(m[1]), floating=int(m[2]), n_q=int(m[3]), n_qd=int(m[4]), n_geoms=int(m[5]),
                n_vis=int(m[6]), has_plane=int(m[7]))


def merge_models(models):
    """A world of several multibodies: the flat models of K fixed-base multibodies (each ONE root link, e.g. the reference's
    `*_xyz_xyzrot.urdf` free-body emulations) -> one flat model with header field TDSM_H_NBODIES = K
    (include/tds_b200_model.h).  Mirrors a reference World holding the plane (if any model has one: multibody 0) and the K
    multibodies in the order given: geoms of different multibodies collide (src/world.hpp:206-282: sphere-sphere,
    capsule-sphere), geoms of one multibody never do; coordinates q / qd are the concatenation in the same order."""
    ms = [np.asarray(m, dtype=np.float64) for m in models]
    if len(ms) < 2:
        raise ValueError("merge_models needs at least two multibodies")
    dims = [model_dims(m) for m in ms]
    if any(d["floating"] for d in dims):
        raise ValueError("merge_models: fixed-base multibodies only (emulate a free body by prismatic + revolute / spherical joints)")
    head = np.zeros(HEADER)
    head[0] = MAGIC
    links, base_geoms, link_geoms, vis = [], [], [], []
    lo = qo = qdo = 0
    for m, d in zip(ms, dims):
        L0 = HEADER + BASE
        G0 = L0 + d["n_links"] * LINK
        V0 = G0 + d["n_geoms"] * GEOM
        l = m[L0:G0].reshape(d["n_links"], LINK).copy()
        if int(np.sum(l[:, 0] < 0)) != 1:
            raise ValueError("merge_models: every multibody must have exactly one root link")
        l[:, 0] = np.where(l[:, 0] >= 0, l[:, 0] + lo, -1)
        moving = l[:, 1] >= 0          # JOINT_FIXED = -1 carries no coordinate
        l[moving, 2] += qo
        l[moving, 3] += qdo
        links.append(l)
        g = m[G0:V0].reshape(d["n_geoms"], GEOM).copy()
        base_geoms.append(g[g[:, 0] < 0])
        gl = g[g[:, 0] >= 0]
        gl[:, 0] += lo
        link_geoms.append(gl)
        v = m[V0:V0 + d["n_vis"] * VIS].reshape(d["n_vis"], VIS).copy()
        v[:, 0] = np.where(v[:, 0] >= 0, v[:, 0] + lo, -1)
        vis.append(v)
        lo += d["n_links"]; qo += d["n_q"]; qdo += d["n_qd"]
        if d["has_plane"] and not head[7]:
            head[7] = 1
            head[8:12] = m[8:12]
    geoms = np.concatenate(base_geoms + link_geoms) if (base_geoms or link_geoms) else np.zeros((0, GEOM))
    vis = np.concatenate(vis) if vis else np.zeros((0, VIS))
    head[1], head[2], head[3], head[4], head[5], head[6], head[12] = lo, 0, qo, qdo, len(geoms), len(vis), len(ms)
    return np.concatenate([head, ms[0][HEADER:HEADER + BASE], np.concatenate(links).ravel(), geoms.ravel(), vis.ravel()])


_BODY_COMPONENTS = ("mass", "com.x", "com.y", "com.z", "inertia.xx", "inertia.xy", "inertia.xz", "inertia.yy", "inertia.yz", "inertia.zz")
_INERTIA_SYM = ((0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2))
# World::default_friction / default_restitution of the reference (src/world.hpp), the simulator's defaults (BatchSim.set_params)
DEFAULT_FRICTION, DEFAULT_RESTITUTION = 0.5, 0.0


def param_names(model):
    """Names of the physical parameter ids of a flat model (include/tds_b200.h), index = id: "friction", "restitution",
    "base.mass", "base.com.x", ..., "link<i>.inertia.zz", then "link<i>.stiffness", "link<i>.damping".  Base ids exist for
    fixed-base models too (they cannot be installed there).  Host only."""
    n_links = model_dims(model)["n_links"]
    names = ["friction", "restitution"]
    for b in range(n_links + 1):
        body = "base" if b == 0 else f"link{b - 1}"
        names += [f"{body}.{c}" for c in _BODY_COMPONENTS]
    for i in range(n_links):
        names += [f"link{i}.stiffness", f"link{i}.damping"]
    return names


def param_values(model, friction=DEFAULT_FRICTION, restitution=DEFAULT_RESTITUTION):
    """The model's value of every parameter id (float64, index = id): friction and restitution are the solver settings given
    (the simulator's defaults unless stated), off-diagonal inertias the symmetric component 0.5 (I_ab + I_ba) the model compiler
    uses.  Host only."""
    m = np.asarray(model, dtype=np.float64)
    n_links = model_dims(m)["n_links"]
    out = [float(friction), float(restitution)]
    for b in range(n_links + 1):
        rec = m[HEADER:HEADER + BASE] if b == 0 else m[HEADER + BASE + (b - 1) * LINK + 19:HEADER + BASE + (b - 1) * LINK + 32]
        inertia = rec[4:13].reshape(3, 3)
        out += list(rec[0:4]) + [0.5 * (inertia[r, c] + inertia[c, r]) for r, c in _INERTIA_SYM]
    for i in range(n_links):
        rec = m[HEADER + BASE + i * LINK:HEADER + BASE + (i + 1) * LINK]
        out += [rec[32], rec[33]]
    return np.asarray(out, dtype=np.float64)


def param_ids(model, names_or_ids):
    """Parameter names and / or ids -> list of int ids (ValueError for an unknown name)."""
    names = None
    ids = []
    for x in names_or_ids:
        if isinstance(x, str):
            names = names or {nm: k for k, nm in enumerate(param_names(model))}
            if x not in names:
                raise ValueError(f"unknown physical parameter {x!r}")
            ids.append(names[x])
        else:
            ids.append(int(x))
    return ids


def set_param_values(model, ids, values):
    """A copy of the flat model with parameter ids (not friction / restitution: those are solver settings) set to values, as
    the simulator applies them per environment; an off-diagonal inertia id sets both entries."""
    m = np.array(model, dtype=np.float64)
    n_links = model_dims(m)["n_links"]
    j0 = 2 + 10 * (n_links + 1)
    for i, v in zip(ids, values):
        if i < 2:
            raise ValueError("friction / restitution are solver settings, not model entries")
        if i < j0:
            b, c = divmod(i - 2, 10)
            o = HEADER if b == 0 else HEADER + BASE + (b - 1) * LINK + 19
            if c < 4:
                m[o + c] = v
            else:
                r, cc = _INERTIA_SYM[c - 4]
                m[o + 4 + 3 * r + cc] = v
                m[o + 4 + 3 * cc + r] = v
        else:
            li, c = divmod(i - j0, 2)
            m[HEADER + BASE + li * LINK + 32 + c] = v
    return m


_REGRESSOR_COMPONENTS = ("m", "mcx", "mcy", "mcz", "Ixx", "Ixy", "Ixz", "Iyy", "Iyz", "Izz")


def regressor_names(model):
    """One name per column of the regressors (BatchSim.regressor_host, DESIGN.md section 7.19): "base.m", "base.mcx", ...,
    "link<i>.Izz" (mass, first moment m c and inertia about the body-frame origin of each body), then "link<i>.stiffness",
    "link<i>.damping".  Column j is physical-parameter id j + 2.  Host only."""
    n_links = model_dims(model)["n_links"]
    names = []
    for b in range(n_links + 1):
        body = "base" if b == 0 else f"link{b - 1}"
        names += [f"{body}.{c}" for c in _REGRESSOR_COMPONENTS]
    for i in range(n_links):
        names += [f"link{i}.stiffness", f"link{i}.damping"]
    return names


def inertial_parameters(model, ids=None, values=None):
    """The regressors' parameter vector pi (float64, DESIGN.md section 7.19): [n_pi] from the model's own values, or [n, n_pi] from a
    per-environment set (ids, values [n, k]) laid out as BatchSim.set_physical_params takes it (the other parameters keep the model's
    values).  Body b: [m, m c, I_com + m (|c|^2 1 - c c^T)] (xx, xy, xz, yy, yz, zz), c the centre of mass in the body frame; link i:
    stiffness and damping rounded to fp32, as the step and inverse dynamics read them.  Host only."""
    base = param_values(model)[2:]
    if ids is None:
        theta = base[None, :]
    else:
        vals = np.atleast_2d(np.asarray(values, dtype=np.float64))
        theta = np.repeat(base[None, :], vals.shape[0], axis=0)
        for k, i in enumerate(ids):
            if int(i) < 2:
                raise ValueError("friction / restitution do not enter the regressors")
            theta[:, int(i) - 2] = vals[:, k]
    n_links = model_dims(model)["n_links"]
    pi = theta.copy()
    for b in range(n_links + 1):
        t = theta[:, 10 * b:10 * b + 10]
        m, c = t[:, 0], t[:, 1:4]
        cc = np.sum(c * c, axis=1)
        out = pi[:, 10 * b:10 * b + 10]
        out[:, 1:4] = m[:, None] * c
        for k, (r, s) in enumerate(_INERTIA_SYM):
            out[:, 4 + k] = t[:, 4 + k] + m * ((cc if r == s else 0.0) - c[:, r] * c[:, s])
    j0 = 10 * (n_links + 1)
    pi[:, j0:] = pi[:, j0:].astype(np.float32).astype(np.float64)
    return pi[0] if ids is None else pi


def save_model(path, model, meta=None):
    with open(path, "w") as f:
        json.dump({"layout": "tds_b200_model.h", "meta": meta or {}, "model": [float(v) for v in model]}, f)


def load_model(path):
    with open(path) as f:
        d = json.load(f)
    return np.asarray(d["model"], dtype=np.float64)


def fixture_path(name):
    """Compiled models shipped with the package (`models/<name>.json`: flat models exported from the reference's own URDF
    loader by tests/golden/make_golden.py, which also keeps the copy under tests/golden/models the tests compare against)."""
    here = os.path.dirname(os.path.abspath(__file__))
    p = os.path.join(here, "models", name + ".json")
    if os.path.exists(p):
        return p
    return os.path.join(os.path.dirname(here), "tests", "golden", "models", name + ".json")
