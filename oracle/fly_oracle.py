"""ctypes binding of the CPU oracle (`oracle/fly_oracle.c`).  TEST INFRASTRUCTURE ONLY:
imported by tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from flybody_b200 import abi

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

# field ids: include/flybody_b200.h enum FbField without FB_ (QPOS, QVEL, ...), the names orc_get / orc_set switch on
globals().update({name[3:]: v for name, v in abi.read().enums['FbField'].items()})


def build(force=False):
    so = os.path.join(_HERE, 'libflyoracle.so')
    src = os.path.join(_HERE, 'fly_oracle.c')
    if force or not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        subprocess.check_call(['make', '-C', _HERE, '-s'] + (['-B'] if force else []))
    return so


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
        _LIB.orc_create.restype = C.c_void_p
        _LIB.orc_create.argtypes = [C.c_void_p]
        for fn in ('orc_destroy', 'orc_step1', 'orc_step2', 'orc_forward', 'orc_step'):
            getattr(_LIB, fn).argtypes = [C.c_void_p]
            getattr(_LIB, fn).restype = None
        _LIB.orc_control_step.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        _LIB.orc_reset.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        _LIB.orc_get.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        _LIB.orc_set.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        _LIB.orc_set_tolerance.argtypes = [C.c_void_p, C.c_double]
        _LIB.orc_set_dense.argtypes = [C.c_void_p, C.c_int]
        _LIB.orc_get_efc.argtypes = [C.c_void_p] + [C.c_void_p] * 6
        _LIB.orc_pair.argtypes = [C.c_int] + [C.c_void_p] * 3 + [C.c_int] + [C.c_void_p] * 3 + [C.c_double, C.c_void_p]
    return _LIB


def pair(t1, p1, R1, s1, t2, p2, R2, s2, margin):
    """one geom pair through the collision stage's narrowphase (no broadphase; a plane is t1 = 0 with its normal the third column of
    R1): the contacts as rows [n, 13] of dist, pos[3], frame[9] (normal, first tangent, second tangent)"""
    d = [np.ascontiguousarray(x, np.float64).ravel() for x in (p1, R1, s1, p2, R2, s2)]
    out = np.zeros((4, 13), np.float64)
    n = lib().orc_pair(int(t1), *[x.ctypes.data for x in d[:3]], int(t2), *[x.ctypes.data for x in d[3:]], float(margin),
                       out.ctypes.data)
    return out[:n].copy()


class Oracle:
    """One double-precision environment stepped by the restated pipeline."""

    def __init__(self, model, tolerance=None, dense=False):
        """dense=True: the original dense statement (Cholesky of M, of M + hD and of the Newton Hessian); default: MuJoCo's
        tree-sparse L^T D L for M and the low-rank form of the Newton Hessian -- same numbers to round-off, ~5x faster."""
        self.model = model
        self._l = lib()
        self._d = self._l.orc_create(C.byref(model.c))
        if not self._d:
            raise ValueError('orc_create refused the model: an actuator has a dynamics or bias type the oracle does not implement '
                             '(dyntype none / filter, biastype none / affine) or an activation address that does not match its dyntype, '
                             'or a touch sensor is on a site that is neither a sphere nor a capsule')
        self._l.orc_set_dense(self._d, 1 if dense else 0)
        if tolerance is not None:
            self._l.orc_set_tolerance(self._d, float(tolerance))
        self._buf = np.zeros(max(model.nv * model.nv, 16 * 64, 9 * model.nbody, 1024), np.float64)

    def __del__(self):
        try:
            self._l.orc_destroy(self._d)
        except Exception:
            pass

    def set_hfield(self, geom, size, heights, pair_geom):
        """terrain for the collision stage: heights [nrow, ncol] as fractions of the elevation scale size[2]."""
        h = np.ascontiguousarray(heights, np.float64); sz = np.ascontiguousarray(size, np.float64); pg = np.ascontiguousarray(pair_geom, np.int32)
        self._l.orc_set_hfield.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int]
        self._l.orc_set_hfield.restype = None
        self._l.orc_set_hfield(self._d, int(geom), sz.ctypes.data, h.shape[0], h.shape[1], h.ctypes.data, pg.ctypes.data, len(pg))

    def get(self, field):
        n = self._l.orc_get(self._d, field, self._buf.ctypes.data)
        if n < 0:
            raise KeyError(field)
        return self._buf[:n].copy()

    def set(self, field, v):
        v = np.ascontiguousarray(v, dtype=np.float64)
        if self._l.orc_set(self._d, field, v.ctypes.data) != 0:
            raise KeyError(field)

    def reset(self, qpos=None, qvel=None):
        qp = None if qpos is None else np.ascontiguousarray(qpos, np.float64)
        qv = None if qvel is None else np.ascontiguousarray(qvel, np.float64)
        self._l.orc_reset(self._d, None if qp is None else qp.ctypes.data, None if qv is None else qv.ctypes.data)

    def forward(self):
        self._l.orc_forward(self._d)

    def step1(self):
        self._l.orc_step1(self._d)

    def step2(self):
        self._l.orc_step2(self._d)

    def step(self):
        self._l.orc_step(self._d)

    def control_step(self, nsub):
        out = np.zeros(self.model.nsensordata, np.float64)
        self._l.orc_control_step(self._d, int(nsub), out.ctypes.data)
        return out

    def efc(self):
        nv = self.model.nv
        J = np.zeros((600, nv)); aref = np.zeros(600); D = np.zeros(600); R = np.zeros(600); pos = np.zeros(600)
        tp = np.zeros(600, np.int32)
        n = self._l.orc_get_efc(self._d, J.ctypes.data, aref.ctypes.data, D.ctypes.data, R.ctypes.data,
                                pos.ctypes.data, tp.ctypes.data)
        return dict(J=J[:n], aref=aref[:n], D=D[:n], R=R[:n], pos=pos[:n], type=tp[:n])

    # convenience
    @property
    def qpos(self):
        return self.get(QPOS)

    @property
    def qvel(self):
        return self.get(QVEL)

    @property
    def qacc(self):
        return self.get(QACC)
