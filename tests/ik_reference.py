"""ctypes binding of tests/ik_reference.c, the fp64 restatement of the reference's qpos_from_site_xpos loop the IK tests and
tools/gpu_ik.py compare the CUDA solver against.  TEST INFRASTRUCTURE ONLY.  The library is compiled on first use into a temporary
directory (the repository tree may be read-only where the tests run)."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


class IkProblem(C.Structure):
    _fields_ = [('n_sites', C.c_int), ('site_ids', C.c_void_p), ('n_jnts', C.c_int), ('jnt_ids', C.c_void_p), ('include', C.c_void_p),
                ('target', C.c_void_p), ('reg', C.c_double), ('lr', C.c_double), ('beta', C.c_double), ('thr', C.c_double),
                ('max_steps', C.c_int)]


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(tempfile.mkdtemp(prefix='ikref_'), 'libikref.so')
        subprocess.check_call([os.environ.get('CC', 'gcc'), '-O2', '-std=c11', '-fPIC', '-shared', '-o', so,
                               os.path.join(_HERE, 'ik_reference.c'), '-lm'])
        _LIB = C.CDLL(so)
        _LIB.ikref_objective.argtypes = [C.c_void_p] * 4
        _LIB.ikref_objective.restype = C.c_double
        _LIB.ikref_solve.argtypes = [C.c_void_p] * 7
    return _LIB


def _problem(site_ids, jnt_ids, target, include, reg_strength, lr, beta, progress_threshold, max_steps):
    keep = [np.ascontiguousarray(site_ids, np.int32).reshape(-1), np.ascontiguousarray(jnt_ids, np.int32).reshape(-1),
            np.ascontiguousarray(target, np.float64).reshape(-1),
            None if include is None else np.ascontiguousarray(include, np.uint8).reshape(-1)]
    p = IkProblem(len(keep[0]), keep[0].ctypes.data, len(keep[1]), keep[1].ctypes.data, None if keep[3] is None else keep[3].ctypes.data,
                  keep[2].ctypes.data, float(reg_strength), float(lr), float(beta), float(progress_threshold), int(max_steps))
    return p, keep


def objective(model, qpos, site_ids, jnt_ids, target, include=None, reg_strength=0.0):
    """(objective, gradient over the fitted dofs in joint order) at qpos"""
    p, keep = _problem(site_ids, jnt_ids, target, include, reg_strength, 0, 0, 0, 1)
    q = np.array(qpos, np.float64)
    g = np.zeros(model.nv, np.float64)
    f = lib().ikref_objective(C.byref(model.c), C.byref(p), q.ctypes.data, g.ctypes.data)
    if np.isnan(f):
        raise ValueError('the fp64 IK reference refused the problem')
    n = sum(6 if int(model.jnt_type[j]) == 0 else 1 for j in np.asarray(jnt_ids).reshape(-1))
    return f, g[:n]


def solve(model, qpos, site_ids, jnt_ids, target, include=None, reg_strength=0.0, lr=0.01, beta=0.99, progress_threshold=0.01,
          max_steps=20_000):
    """the reference's loop in fp64 from qpos -> dict(qpos, err_norm, err_norm_first_term, steps, success)"""
    p, keep = _problem(site_ids, jnt_ids, target, include, reg_strength, lr, beta, progress_threshold, max_steps)
    q = np.array(qpos, np.float64)
    err, err1, steps, ok = C.c_double(), C.c_double(), C.c_int(), C.c_int()
    if lib().ikref_solve(C.byref(model.c), C.byref(p), q.ctypes.data, C.byref(err), C.byref(err1), C.byref(steps), C.byref(ok)) != 0:
        raise ValueError('the fp64 IK reference refused the problem')
    return dict(qpos=q, err_norm=err.value, err_norm_first_term=err1.value, steps=steps.value, success=bool(ok.value))
