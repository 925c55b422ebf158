"""`import pytinydiffsim` for scripts written against the reference's Python module: the hot-path names
(python/pytinydiffsim.inl) served by libtds_b200.so.  See tds_b200/pytinydiffsim.py."""
from tds_b200.pytinydiffsim import *  # noqa: F401,F403
from tds_b200.pytinydiffsim import (TinyWorld, TinyMultiBody, TinyUrdfParser, TinyUrdfStructures, UrdfToMultiBody2,  # noqa: F401
                                    forward_dynamics, integrate_euler, integrate_euler_qdd, mass_matrix, point_jacobian, inverse_dynamics,
                                    bias_forces, CartpoleEnv,
                                    VectorizedLaikagoEnv, VectorizedAntEnv)
