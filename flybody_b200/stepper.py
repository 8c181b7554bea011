"""ctypes binding of the CUDA stepper's C ABI (`include/flybody_b200.h`; its prototypes, enums and program structs are read from
the header by `abi.py`).

`BatchedStepper` is the batched stand-in for the `physics` object that dm_control hands to the
reference's task hooks (SURVEY.md 8(b)): `set_control`, `step`, state reads.  It fails loudly
when the CUDA library is missing -- there is no CPU fallback in the product path.
"""
import ctypes as C
import os

import numpy as np

from . import abi
from .abi import StepperError
from .flymodel import FlyModel

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'lib', 'libflybody_b200.so')

_ABI = abi.read()
# enum FbField (fb_get / fb_set fields: QPOS .. XFRC_APPLIED), enum FbObsItem (OBS_*), enum FbTaskKind (TASK_*, FbTaskProgram.kind)
# and enum FbSidQuery (SID_TRANSITION, SID_INVERSE), by their header names without FB_
globals().update({name[3:]: v for enum in ('FbField', 'FbObsItem', 'FbTaskKind', 'FbSidQuery') for name, v in _ABI.enums[enum].items()})
MAXCON, MAXEFC = _ABI.defines['FB_MAXCON'], _ABI.defines['FB_MAXEFC']

# enum FbParam: the per-env model parameters (fb_param_*), by their mjModel names, in id order
PARAMS = tuple(name[5:].lower() for name, _ in sorted(_ABI.enums['FbParam'].items(), key=lambda e: e[1]) if name != 'FB_NPARAMS')
FD_ELEMENT, FD_SCALE = 0, 1           # kinds of a parameter direction (fb_fd_param_program)

# the programs of fb_obs_program, fb_task_program, fb_eye_program, fb_ik_program and fb_plan_program
FbObsProgram, FbTaskProgram, FbEyeProgram, FbIkProgram, FbPlanProgram = (_ABI.structs[n] for n in ('FbObsProgram', 'FbTaskProgram',
                                                                                                     'FbEyeProgram', 'FbIkProgram',
                                                                                                     'FbPlanProgram'))


def load_library(path=None):
    """the stepper library with every function the header declares bound to its prototype"""
    path = path or os.environ.get('FLYBODY_B200_LIB') or LIB_PATH      # the env override is for A/B timing of kernel variants
    if not os.path.exists(path):
        raise StepperError(
            f'CUDA stepper library not found at {path}. Build it with `python -c "import __graft_entry__ as g; '
            f'g.build()"` (nvcc, sm_90a). There is no CPU fallback.')
    lib = C.CDLL(path)
    for name, (restype, argtypes) in _ABI.functions.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = restype, argtypes
    return lib


def _batched(model, inputs, run, per, n_envs=None, setup=None, device=0, lib_path=None):
    """The shell of the batched device front ends.  inputs: [(name, array, row shape)], coerced to fp64 rows; the first one without
    its batch dimension makes a single problem.  One handle of n_envs envs (default: min(B, per)) solves `per` problems at a time:
    setup(sim) once, then run(sim, chunk rows, k) -> a tuple of [k, ...] outputs (a list: per-problem objects).
    -> (single, the outputs over all B problems)"""
    rows = [np.asarray(x, np.float64) for _, x, _ in inputs]
    single = rows[0].ndim == len(inputs[0][2])
    B = rows[0].reshape((-1,) + tuple(inputs[0][2])).shape[0]
    rows = [x.reshape((-1 if np.prod(shape) else B,) + tuple(shape)) for x, (_, _, shape) in zip(rows, inputs)]
    if any(x.shape[0] != B for x in rows):
        raise ValueError(', '.join(f'{x.shape[0]} {name} rows' for x, (name, _, _) in zip(rows, inputs)))
    sim = BatchedStepper(model, min(B, per) if n_envs is None else n_envs, device=device, lib_path=lib_path)
    outs = []
    try:
        if setup is not None:
            setup(sim)
        for p0 in range(0, B, per):
            k = min(per, B - p0)
            outs.append(run(sim, [x[p0:p0 + k] for x in rows], k))
    finally:
        sim.close()
    return single, [np.concatenate(c) if isinstance(c[0], np.ndarray) else [x for part in c for x in part] for c in zip(*outs)]


class BatchedStepper:
    """N fly environments stepped in lock-step on one device."""

    def __init__(self, model: FlyModel, n_envs: int, device: int = 0, lib_path: str | None = None):
        self.model = model
        self.n_envs = int(n_envs)
        self.device = int(device)
        self._lib = load_library(lib_path)
        h = C.c_void_p()
        rc = self._lib.fb_create(C.byref(model.c), self.n_envs, int(device), C.byref(h))
        self._h = h
        if rc != 0:
            msg = self._lib.fb_last_error(h).decode() if h else 'no handle'
            raise StepperError(f'fb_create failed ({rc}): {msg}')

    def close(self):
        if getattr(self, '_h', None):
            self._lib.fb_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc, what):
        if rc != 0:
            raise StepperError(f'{what} failed ({rc}): {self._lib.fb_last_error(self._h).decode()}')

    # -- state access ---------------------------------------------------------------------
    def get(self, field):
        n = self._lib.fb_field_size(self._h, field)
        if n < 0:
            raise KeyError(field)
        out = np.zeros((self.n_envs, max(n, 1)), np.float32)
        self._check(self._lib.fb_get(self._h, field, out.ctypes.data, 0), 'fb_get')
        return out[:, :n]

    def set(self, field, values):
        v = np.ascontiguousarray(np.broadcast_to(np.asarray(values, np.float32), (self.n_envs, np.asarray(values).shape[-1])))
        self._check(self._lib.fb_set(self._h, field, v.ctypes.data), 'fb_set')

    def set_control(self, ctrl):
        """physics.set_control (reference fruitfly.py:540-544), ctrl [N, nu] (or [nu], broadcast)."""
        k = getattr(self, '_n_ctrl_cols', self.model.nu)      # action columns after set_action_map, else nu
        c = np.ascontiguousarray(np.broadcast_to(np.asarray(ctrl, np.float32), (self.n_envs, k)))
        self._check(self._lib.fb_set_ctrl(self._h, c.ctypes.data, 0), 'fb_set_ctrl')

    def write_state(self, field, idx, vals):
        idx = np.ascontiguousarray(idx, np.int32)
        v = np.ascontiguousarray(np.broadcast_to(np.asarray(vals, np.float32), (self.n_envs, len(idx))))
        self._check(self._lib.fb_write_state(self._h, field, idx.ctypes.data, len(idx), v.ctypes.data), 'fb_write_state')

    # ---- applied forces (mjData.qfrc_applied / xfrc_applied; persist until overwritten, zeroed by a reset of the env)
    def set_applied(self, qfrc=None, xfrc=None, env_ids=None):
        """qfrc [N or n, nv] generalized forces and / or xfrc [N or n, nbody, 6] world-frame force, then torque, at each body's CoM,
        for every env (env_ids None; rows broadcast) or only the listed envs (the others keep theirs).  None leaves a field as is."""
        for field, v, shape in ((QFRC_APPLIED, qfrc, (self.model.nv,)), (XFRC_APPLIED, xfrc, (self.model.nbody, 6))):
            if v is None:
                continue
            v = np.asarray(v, np.float32)
            if env_ids is None:
                full = np.broadcast_to(v.reshape((-1,) + shape), (self.n_envs,) + shape)
            else:
                ids = np.asarray(env_ids, np.int64).reshape(-1)
                full = self.get(field).reshape((self.n_envs,) + shape)
                full[ids] = np.broadcast_to(v.reshape((-1,) + shape), (len(ids),) + shape)
            self.set(field, np.ascontiguousarray(full).reshape(self.n_envs, -1))

    def applied(self):
        """-> (qfrc_applied [N, nv], xfrc_applied [N, nbody, 6]); zero while unset."""
        return self.get(QFRC_APPLIED), self.get(XFRC_APPLIED).reshape(self.n_envs, self.model.nbody, 6)

    def applied_ptrs(self):
        """(qfrc_applied, xfrc_applied) device pointers of contiguous fp32 rows [N, nv], [N, nbody, 6] to write in place."""
        q, x = C.c_void_p(), C.c_void_p()
        self._check(self._lib.fb_applied_ptrs(self._h, C.byref(q), C.byref(x)), 'fb_applied_ptrs')
        return q.value, x.value

    def clear_applied(self):
        """drop every env's applied forces: the step goes back to the path without them"""
        self._check(self._lib.fb_clear_applied(self._h), 'fb_clear_applied')

    # ---- per-env model parameters (fb_param_*: physics.model writes without mj_setConst, per env; see the header)
    def _param(self, name):
        if name not in PARAMS:
            raise KeyError(f'{name!r} is not a per-env model parameter ({", ".join(PARAMS)})')
        p = PARAMS.index(name)
        return p, int(self._lib.fb_param_size(self._h, p))

    def param_set(self, name, vals, env_ids=None):
        """vals [n_envs or len(env_ids), size] (a [size] row broadcasts) -> every env (env_ids None) or the listed ones"""
        p, k = self._param(name)
        ids = None if env_ids is None else np.ascontiguousarray(np.asarray(env_ids).reshape(-1), np.int32)
        n = self.n_envs if ids is None else len(ids)
        v = np.ascontiguousarray(np.broadcast_to(np.asarray(vals, np.float32).reshape(-1, k), (n, k)))
        self._check(self._lib.fb_param_set(self._h, p, None if ids is None else ids.ctypes.data, n, v.ctypes.data, 0), 'fb_param_set')

    def param_get(self, name):
        """-> [n_envs, size] f32 (the compiled values while there is no overlay)"""
        p, k = self._param(name)
        out = np.zeros((self.n_envs, k), np.float32)
        self._check(self._lib.fb_param_get(self._h, p, out.ctypes.data, 0), 'fb_param_get')
        return out

    def param_draws(self, name, lo=None, hi=None, shared=False, seed=0):
        """draw `name` from [lo, hi] ([size] each, broadcast) at every reset of an env; lo = hi = None stops drawing it"""
        p, k = self._param(name)
        if lo is None and hi is None:
            self._check(self._lib.fb_param_draws(self._h, p, None, None, 0, int(seed)), 'fb_param_draws')
            return
        lo = np.ascontiguousarray(np.broadcast_to(np.asarray(lo, np.float32).reshape(-1), (k,)))
        hi = np.ascontiguousarray(np.broadcast_to(np.asarray(hi, np.float32).reshape(-1), (k,)))
        self._check(self._lib.fb_param_draws(self._h, p, lo.ctypes.data, hi.ctypes.data, int(bool(shared)), int(seed) & 0xffffffff),
                    'fb_param_draws')

    def param_clear(self):
        """drop every env's parameters and the draw program: the step goes back to the compiled model's tables"""
        self._check(self._lib.fb_param_clear(self._h), 'fb_param_clear')

    # ---- state rows (fb_state_*: physics.get_state / set_state for the envs of the batch, see the header)
    @property
    def state_slots(self):
        """4-byte slots of one state row under the current programs"""
        return int(self._lib.fb_state_slots(self._h))

    def state_signature(self):
        """hash of the row layout; rows move between steppers with equal signatures"""
        return int(self._lib.fb_state_signature(self._h))

    def state_bank(self, n_slots):
        """(re)allocate the device bank of `n_slots` state rows (0 frees it)"""
        self._check(self._lib.fb_state_bank(self._h, int(n_slots)), 'fb_state_bank')

    @staticmethod
    def _id_pair(a, b):
        a = None if a is None else np.ascontiguousarray(np.asarray(a).reshape(-1), np.int32)
        b = None if b is None else np.ascontiguousarray(np.asarray(b).reshape(-1), np.int32)
        if a is not None and b is not None and len(a) != len(b):
            raise ValueError(f'{len(a)} ids against {len(b)}')
        n = len(a) if a is not None else (len(b) if b is not None else 0)
        return a, b, n, None if a is None else a.ctypes.data, None if b is None else b.ctypes.data

    def save_state(self, slots=None, env_ids=None):
        """env_ids[k] -> bank slot slots[k] (None: 0 .. n - 1; both None: every env k -> slot k); stream-ordered"""
        e, s, n, ep, sp = self._id_pair(env_ids, slots)
        self._keep_ids = (e, s)
        self._check(self._lib.fb_state_save(self._h, ep, sp, n), 'fb_state_save')

    def load_state(self, slots=None, env_ids=None):
        """bank slot slots[k] -> env env_ids[k] (None: 0 .. n - 1; both None: slot k -> every env k); one slot may feed many envs"""
        s, e, n, sp, ep = self._id_pair(slots, env_ids)
        self._keep_ids = (e, s)
        self._check(self._lib.fb_state_load(self._h, sp, ep, n), 'fb_state_load')

    def read_states(self, slots):
        """-> uint32 [len(slots), state_slots]: the listed bank rows on the host (raw bits)"""
        s = np.ascontiguousarray(np.asarray(slots).reshape(-1), np.int32)
        out = np.zeros((len(s), self.state_slots), np.uint32)
        self._check(self._lib.fb_state_read(self._h, s.ctypes.data, len(s), out.ctypes.data), 'fb_state_read')
        return out

    def write_states(self, slots, rows):
        """host rows (as read_states returns them, of a stepper with the same state_signature) -> the listed bank slots"""
        s = np.ascontiguousarray(np.asarray(slots).reshape(-1), np.int32)
        r = np.ascontiguousarray(rows, np.uint32)
        if r.shape != (len(s), self.state_slots):
            raise ValueError(f'rows {r.shape} against {(len(s), self.state_slots)}')
        self._check(self._lib.fb_state_write(self._h, s.ctypes.data, len(s), r.ctypes.data), 'fb_state_write')

    def state_substeps(self, n_substeps=0):
        """substeps of the last control step (the divisor of the per-step sensor means); a positive argument sets it first"""
        return int(self._lib.fb_state_substeps(self._h, int(n_substeps)))

    # ---- multi-site inverse kinematics (fb_ik_*; flybody_b200.inverse_kinematics is the reference-shaped front end)
    def ik_program(self, site_ids, jnt_ids, include=None, reg_strength=0.0, lr=0.01, beta=0.99, progress_threshold=0.01, max_steps=20_000):
        """fit the listed joints (hinge / free) to the listed sites; include: [3 * n_sites] component mask (None: all)"""
        sid = np.ascontiguousarray(site_ids, np.int32).reshape(-1)
        jid = np.ascontiguousarray(jnt_ids, np.int32).reshape(-1)
        inc = None if include is None else np.ascontiguousarray(include, np.uint8).reshape(-1)
        if inc is not None and len(inc) != 3 * len(sid):
            raise ValueError(f'include has {len(inc)} entries for {len(sid)} sites')
        p = FbIkProgram(len(sid), sid.ctypes.data_as(C.POINTER(C.c_int32)), len(jid), jid.ctypes.data_as(C.POINTER(C.c_int32)),
                        None if inc is None else inc.ctypes.data_as(C.POINTER(C.c_uint8)), float(reg_strength), float(lr), float(beta),
                        float(progress_threshold), int(max_steps))
        self._check(self._lib.fb_ik_program(self._h, C.byref(p)), 'fb_ik_program')
        self._ik_nsite = len(sid)

    def ik_solve(self, target_xpos, init_qpos=None):
        """solve problems 0 .. n-1 (envs) for targets [n, n_sites, 3] from init_qpos [n, nq] (None: the envs' current qpos)"""
        t = np.ascontiguousarray(target_xpos, np.float32).reshape(-1, self._ik_nsite, 3)
        n = t.shape[0]
        q = None if init_qpos is None else np.ascontiguousarray(np.broadcast_to(np.asarray(init_qpos, np.float32), (n, self.model.nq)))
        self._check(self._lib.fb_ik_solve(self._h, n, t.ctypes.data, None if q is None else q.ctypes.data), 'fb_ik_solve')
        self._ik_n = n

    def ik_read(self):
        """-> (qpos [n, nq] f32, err_norm [n] f32, err_norm_first_term [n] f32, steps [n] i32, success [n] bool) of the last solve"""
        n = self._ik_n
        q, e, e1 = np.zeros((n, self.model.nq), np.float32), np.zeros(n, np.float32), np.zeros(n, np.float32)
        k, ok = np.zeros(n, np.int32), np.zeros(n, np.uint8)
        self._check(self._lib.fb_ik_read(self._h, q.ctypes.data, e.ctypes.data, e1.ctypes.data, k.ctypes.data, ok.ctypes.data), 'fb_ik_read')
        return q, e, e1, k, ok.astype(bool)

    # ---- inverse dynamics (fb_inverse; flybody_b200.inverse_dynamics is the batched front end)
    def _problem_rows(self, inputs, n, is_device):
        """the inputs [(name, array or device pointer, row width)] of a call on problems 0 .. n-1 -> (n, pointers, host rows): device
        pointers (ints) with is_device=True and n given, or host arrays of equal row counts as fp32 rows (keep them alive for the call)"""
        if is_device:
            if n is None:
                raise ValueError('device inputs need n')
            return int(n), [C.c_void_p(int(x)) for _, x, _ in inputs], None
        rows = [np.ascontiguousarray(np.asarray(x, np.float32).reshape(-1, k)) for _, x, k in inputs]
        if len({r.shape[0] for r in rows}) != 1:
            raise ValueError(', '.join(f'{r.shape[0]} {name} rows' for (name, _, _), r in zip(inputs, rows)))
        n = rows[0].shape[0] if n is None else int(n)
        if n > rows[0].shape[0]:
            raise ValueError(f'{rows[0].shape[0]} rows for n = {n}')
        return n, [r.ctypes.data for r in rows], rows

    def inverse(self, qacc, n=None, is_device=False):
        """mj_inverse for envs 0 .. n-1 at their current qpos / qvel: qacc [n, nv] (host array), or a device pointer (int) with
        is_device=True and n given.  Stream-ordered; read the results with inverse_read()."""
        n, ptrs, _rows = self._problem_rows([('qacc', qacc, self.model.nv)], n, is_device)
        self._check(self._lib.fb_inverse(self._h, n, *ptrs, int(bool(is_device))), 'fb_inverse')
        self._inv_n = n

    def inverse_read(self):
        """-> (qfrc_inverse [n, nv], qfrc_constraint [n, nv], efc_force [n, MAXEFC]) f32 of the last inverse"""
        n, nv = getattr(self, '_inv_n', 0), self.model.nv
        qi, qc, f = np.zeros((n, nv), np.float32), np.zeros((n, nv), np.float32), np.zeros((n, MAXEFC), np.float32)
        self._check(self._lib.fb_inverse_read(self._h, qi.ctypes.data, qc.ctypes.data, f.ctypes.data, 0), 'fb_inverse_read')
        return qi, qc, f

    # ---- finite-difference transition Jacobians (fb_fd_*; flybody_b200.derivatives is the batched front end)
    def fd_columns(self, centered=True):
        """envs one problem of fd_transition takes"""
        return int(self._lib.fb_fd_columns(self._h, int(bool(centered))))

    def fd_transition(self, slots, eps=1e-2, centered=True, n_substeps=1):
        """A = dx'/dx, B = dx'/du of the bank rows `slots` over n_substeps substeps (see the header); the envs' states are a workspace
        afterwards.  Read the results with fd_read()."""
        s = np.ascontiguousarray(np.asarray(slots).reshape(-1), np.int32)
        self._check(self._lib.fb_fd_transition(self._h, s.ctypes.data, len(s), float(eps), int(bool(centered)), int(n_substeps)),
                    'fb_fd_transition')
        self._fd_n = len(s)

    def fd_read(self):
        """-> (A [n, nx, nx], B [n, nx, nu], qpos_next [n, nq], qvel_next [n, nv], act_next [n, na]) f32 of the last fd_transition"""
        m, n = self.model, getattr(self, '_fd_n', 0)
        nx = 2 * m.nv + m.na
        A, B = np.zeros((n, nx, nx), np.float32), np.zeros((n, nx, m.nu), np.float32)
        q, v, a = np.zeros((n, m.nq), np.float32), np.zeros((n, m.nv), np.float32), np.zeros((n, m.na), np.float32)
        self._check(self._lib.fb_fd_read(self._h, A.ctypes.data, B.ctypes.data, q.ctypes.data, v.ctypes.data, a.ctypes.data, 0), 'fb_fd_read')
        return A, B, q, v, a

    # ---- finite-difference inverse-dynamics Jacobians (fb_fd_inverse*; flybody_b200.derivatives.inverse_fd is the batched front end)
    def fd_inverse_columns(self, centered=True):
        """envs one problem of fd_inverse takes"""
        return int(self._lib.fb_fd_inverse_columns(self._h, int(bool(centered))))

    def fd_inverse(self, qpos, qvel, qacc, eps=1e-2, centered=True, n=None, is_device=False):
        """the Jacobians of qfrc_inverse (and qM) of problems qpos [n, nq], qvel [n, nv], qacc [n, nv] (host arrays), or of device
        pointers (ints) with is_device=True and n given (see the header); the envs' states are a workspace afterwards.  Read the results
        with fd_inverse_read()."""
        m = self.model
        n, ptrs, _rows = self._problem_rows([('qpos', qpos, m.nq), ('qvel', qvel, m.nv), ('qacc', qacc, m.nv)], n, is_device)
        self._check(self._lib.fb_fd_inverse(self._h, n, *ptrs, float(eps), int(bool(centered)), int(bool(is_device))), 'fb_fd_inverse')
        self._fdi_n = n

    def fd_inverse_read(self):
        """-> (DfDq, DfDv, DfDa [n, nv, nv], DmDq [n, nv, nM], qfrc_inverse [n, nv]) f32 of the last fd_inverse, transposed as MuJoCo's:
        DfDq[p, i, j] = d qfrc_inverse_j / d dq_i"""
        m, n = self.model, getattr(self, '_fdi_n', 0)
        out = [np.zeros((n, m.nv, m.nv), np.float32) for _ in range(3)]
        out += [np.zeros((n, m.nv, int(m.nM)), np.float32), np.zeros((n, m.nv), np.float32)]
        self._check(self._lib.fb_fd_inverse_read(self._h, *[x.ctypes.data for x in out], 0), 'fb_fd_inverse_read')
        return tuple(out)

    # ---- sensors in the dynamics queries (fb_query_sensors; see the header)
    def query_sensors(self, on=True):
        """while on, inverse, fd_transition and fd_inverse also produce sensor outputs (read with the *_sensor_read calls)"""
        self._check(self._lib.fb_query_sensors(self._h, int(bool(on))), 'fb_query_sensors')

    def inverse_sensor_read(self):
        """-> sensordata [n, nsd] f32 of the last inverse (run with sensors on)"""
        out = np.zeros((getattr(self, '_inv_n', 0), self.model.nsensordata), np.float32)
        self._check(self._lib.fb_inverse_sensor_read(self._h, out.ctypes.data, 0), 'fb_inverse_sensor_read')
        return out

    def fd_sensor_read(self):
        """-> (C [n, nsd, nx], D [n, nsd, nu], sensordata [n, nsd]) f32 of the last fd_transition (run with sensors on): the sensors
        of the state before the step and their derivatives"""
        m, n = self.model, getattr(self, '_fd_n', 0)
        nsd = m.nsensordata
        out = [np.zeros((n, nsd, 2 * m.nv + m.na), np.float32), np.zeros((n, nsd, m.nu), np.float32), np.zeros((n, nsd), np.float32)]
        self._check(self._lib.fb_fd_sensor_read(self._h, *[x.ctypes.data for x in out], 0), 'fb_fd_sensor_read')
        return tuple(out)

    def fd_inverse_sensor_read(self):
        """-> (DsDq, DsDv, DsDa [n, nv, nsd], sensordata [n, nsd]) f32 of the last fd_inverse (run with sensors on), transposed as
        MuJoCo's: DsDq[p, i, k] = d sensordata_k / d dq_i"""
        m, n = self.model, getattr(self, '_fdi_n', 0)
        out = [np.zeros((n, m.nv, m.nsensordata), np.float32) for _ in range(3)] + [np.zeros((n, m.nsensordata), np.float32)]
        self._check(self._lib.fb_fd_inverse_sensor_read(self._h, *[x.ctypes.data for x in out], 0), 'fb_fd_inverse_sensor_read')
        return tuple(out)

    # ---- finite-difference parameter Jacobians (fb_fd_param_*; flybody_b200.derivatives.parameter_fd / inverse_parameter_fd are the
    # batched front ends)
    def fd_param_program(self, directions):
        """directions: [(kind, [(parameter name, element), ...], [floor per entry] or None)], kind FD_ELEMENT (one entry) or FD_SCALE;
        an empty list clears the program (see the header)"""
        kind, ptr, par, elem, floor = [], [0], [], [], []
        for k, entries, floors in directions:
            kind.append(int(k))
            for t, (name, i) in enumerate(entries):
                par.append(self._param(name)[0])
                elem.append(int(i))
                floor.append(1.0 if floors is None else float(floors[t]))
            ptr.append(len(par))
        arrs = [np.ascontiguousarray(x, np.int32) for x in (kind, ptr, par, elem)] + [np.ascontiguousarray(floor, np.float32)]
        self._check(self._lib.fb_fd_param_program(self._h, len(kind), *[x.ctypes.data for x in arrs]), 'fb_fd_param_program')
        self._fdp_k = len(kind)

    def fd_param_columns(self, centered=True):
        """envs one problem of fd_param_transition / fd_param_inverse takes"""
        n = int(self._lib.fb_fd_param_columns(self._h, int(bool(centered))))
        self._check(0 if n > 0 else -1, 'fb_fd_param_columns')
        return n

    def fd_param_transition(self, slots, eps=1e-2, centered=True, n_substeps=1):
        """dx'/dtheta of the bank rows `slots` along the program's directions over n_substeps substeps; read with fd_param_read()"""
        s = np.ascontiguousarray(np.asarray(slots).reshape(-1), np.int32)
        self._check(self._lib.fb_fd_param_transition(self._h, s.ctypes.data, len(s), float(eps), int(bool(centered)), int(n_substeps)),
                    'fb_fd_param_transition')
        self._fdp_n = (len(s), self._fdp_k)

    def fd_param_read(self):
        """-> (dxdp [n, nx, k], qpos_next [n, nq], qvel_next [n, nv], act_next [n, na]) f32 of the last fd_param_transition"""
        m, (n, k) = self.model, getattr(self, '_fdp_n', (0, 0))
        out = [np.zeros((n, 2 * m.nv + m.na, k), np.float32), np.zeros((n, m.nq), np.float32), np.zeros((n, m.nv), np.float32),
               np.zeros((n, m.na), np.float32)]
        self._check(self._lib.fb_fd_param_read(self._h, *[x.ctypes.data for x in out], 0), 'fb_fd_param_read')
        return tuple(out)

    def fd_param_sensor_read(self):
        """-> (dsdp [n, nsd, k], sensordata [n, nsd]) f32 of the last fd_param_transition (run with sensors on): the sensors of x"""
        m, (n, k) = self.model, getattr(self, '_fdp_n', (0, 0))
        out = [np.zeros((n, m.nsensordata, k), np.float32), np.zeros((n, m.nsensordata), np.float32)]
        self._check(self._lib.fb_fd_param_sensor_read(self._h, *[x.ctypes.data for x in out], 0), 'fb_fd_param_sensor_read')
        return tuple(out)

    def fd_param_inverse(self, qpos, qvel, qacc, eps=1e-2, centered=True, n=None, is_device=False):
        """d qfrc_inverse / dtheta of problems qpos [n, nq], qvel [n, nv], qacc [n, nv] along the program's directions, problem i with
        env i's parameters (host arrays, or device pointers with is_device=True and n given); read with fd_param_inverse_read()"""
        m = self.model
        n, ptrs, _rows = self._problem_rows([('qpos', qpos, m.nq), ('qvel', qvel, m.nv), ('qacc', qacc, m.nv)], n, is_device)
        self._check(self._lib.fb_fd_param_inverse(self._h, n, *ptrs, float(eps), int(bool(centered)), int(bool(is_device))),
                    'fb_fd_param_inverse')
        self._fdpi_n = (n, self._fdp_k)

    def fd_param_inverse_read(self):
        """-> (DfDp [n, k, nv], qfrc_inverse [n, nv]) f32 of the last fd_param_inverse: DfDp[p, j, i] = d qfrc_inverse_i / d direction j"""
        m, (n, k) = self.model, getattr(self, '_fdpi_n', (0, 0))
        out = [np.zeros((n, k, m.nv), np.float32), np.zeros((n, m.nv), np.float32)]
        self._check(self._lib.fb_fd_param_inverse_read(self._h, *[x.ctypes.data for x in out], 0), 'fb_fd_param_inverse_read')
        return tuple(out)

    def fd_param_inverse_sensor_read(self):
        """-> (DsDp [n, k, nsd], sensordata [n, nsd]) f32 of the last fd_param_inverse (run with sensors on)"""
        m, (n, k) = self.model, getattr(self, '_fdpi_n', (0, 0))
        out = [np.zeros((n, k, m.nsensordata), np.float32), np.zeros((n, m.nsensordata), np.float32)]
        self._check(self._lib.fb_fd_param_inverse_sensor_read(self._h, *[x.ctypes.data for x in out], 0), 'fb_fd_param_inverse_sensor_read')
        return tuple(out)

    # ---- batched rollouts (fb_rollout*; flybody_b200.rollout is the batched front end)
    def _inputs(self, inputs, is_device):
        """[(name, array, shape)] -> (pointers, host fp32 arrays to keep alive); device pointers (ints) pass through with is_device"""
        if is_device:
            return [None if x is None else C.c_void_p(int(x)) for _, x, _ in inputs], None
        keep = [None if x is None else np.ascontiguousarray(np.asarray(x, np.float32)) for _, x, _ in inputs]
        for (name, _, shape), x in zip(inputs, keep):
            if x is not None and x.shape != shape:
                raise ValueError(f'{name} {x.shape} against {shape}')
        return [None if x is None else x.ctypes.data for x in keep], keep

    def rollout_feedback(self, x_ref=None, K=None, T=None, is_device=False):
        """the feedback law of the rollouts that follow: ctrl = ctrl_t + K_t (x_t - x_ref_t), x_ref [T, nq + nv + na], K [T, nu, nx]
        (host arrays, or device pointers with is_device=True and T given); None for both clears it (see the header)"""
        m = self.model
        if x_ref is None and K is None:
            self._check(self._lib.fb_rollout_feedback(self._h, 0, None, None, 0), 'fb_rollout_feedback')
            return
        T = int(T if is_device else np.shape(x_ref)[0])
        ptrs, _keep = self._inputs([('x_ref', x_ref, (T, m.nq + m.nv + m.na)), ('K', K, (T, m.nu, 2 * m.nv + m.na))], is_device)
        self._check(self._lib.fb_rollout_feedback(self._h, T, *ptrs, int(bool(is_device))), 'fb_rollout_feedback')

    def rollout_feedback_bank(self, x_ref, K, law, L=None, T=None, is_device=False):
        """a bank of L feedback laws, x_ref [L, T, nq + nv + na] and K [L, T, nu, nx] (host arrays, or device pointers with is_device=True
        and L, T given), and law [n] (host ints in [0, L)): rollout i of the n-rollout calls that follow applies law law[i]"""
        m = self.model
        if not is_device:
            L, T = np.shape(x_ref)[:2]
        L, T = int(L), int(T)
        lw = np.ascontiguousarray(np.asarray(law).reshape(-1), np.int32)
        ptrs, _keep = self._inputs([('x_ref', x_ref, (L, T, m.nq + m.nv + m.na)), ('K', K, (L, T, m.nu, 2 * m.nv + m.na))], is_device)
        self._check(self._lib.fb_rollout_feedback_bank(self._h, L, T, *ptrs, lw.ctypes.data, len(lw), int(bool(is_device))),
                    'fb_rollout_feedback_bank')

    def rollout(self, slots, ctrl, n_substeps=1, qfrc_applied=None, xfrc_applied=None, T=None, is_device=False):
        """rollout i from bank row slots[i] in env i: ctrl [n, T, nu], optional qfrc_applied [n, T, nv] and xfrc_applied [n, T, nbody, 6]
        (host arrays, or device pointers with is_device=True and T given); T control steps of n_substeps substeps.  The envs' states
        are a workspace afterwards.  Read the records with rollout_read()."""
        m = self.model
        s = np.ascontiguousarray(np.asarray(slots).reshape(-1), np.int32)
        n = len(s)
        T = int(T if is_device else np.shape(ctrl)[1])
        ptrs, _keep = self._inputs([('ctrl', ctrl, (n, T, m.nu)), ('qfrc_applied', qfrc_applied, (n, T, m.nv)),
                                    ('xfrc_applied', xfrc_applied, (n, T, m.nbody, 6))], is_device)
        self._check(self._lib.fb_rollout(self._h, s.ctypes.data, n, T, int(n_substeps), *ptrs, int(bool(is_device))), 'fb_rollout')
        self._roll = (n, T)

    def _outputs(self, out, shapes, dtypes):
        """caller-provided outputs (numpy arrays or torch tensors, C-contiguous, of the given shapes and dtypes; None: not read) or new
        numpy arrays -> (arrays, pointers, is_device: a CUDA tensor among them)"""
        if out is None:
            out = [np.zeros(sh, dt) for sh, dt in zip(shapes, dtypes)]
        if len(out) != len(shapes):
            raise ValueError(f'{len(out)} outputs against {len(shapes)}')
        ptrs, dev = [], False
        for x, sh, dt in zip(out, shapes, dtypes):
            if x is None:                                            # an output the caller skips (the ABI's NULL)
                ptrs.append(None)
                continue
            if isinstance(x, np.ndarray):
                ok = x.dtype == dt and x.flags.c_contiguous
                ptrs.append(x.ctypes.data)
            else:                                                    # a torch tensor
                ok = str(x.dtype) == f'torch.{np.dtype(dt).name}' and x.is_contiguous()
                ptrs.append(x.data_ptr())
                dev = dev or x.is_cuda
            if not ok or tuple(x.shape) != tuple(sh):
                raise ValueError(f'output {tuple(x.shape)} {x.dtype} against a contiguous {tuple(sh)} {np.dtype(dt).name}')
        return out, ptrs, dev

    def rollout_read(self, out=None):
        """-> (qpos [n, T, nq], qvel [n, T, nv], act [n, T, na], ctrl [n, T, nu], time [n, T] f32, flags [n, T] i32) of the last
        rollout; out: the six arrays to fill instead (numpy arrays, or torch tensors, CUDA ones by device pointer)"""
        m, (n, T) = self.model, getattr(self, '_roll', (0, 0))
        shapes = [(n, T, m.nq), (n, T, m.nv), (n, T, m.na), (n, T, m.nu), (n, T), (n, T)]
        out, ptrs, dev = self._outputs(out, shapes, [np.float32] * 5 + [np.int32])
        self._check(self._lib.fb_rollout_read(self._h, *ptrs, int(dev)), 'fb_rollout_read')
        return tuple(out)

    def rollout_sensor_read(self, out=None):
        """-> (sensordata [n, T, nsd], sensor_mean [n, T, nsd]) f32 of the last rollout (run with sensors on); out as rollout_read's"""
        m, (n, T) = self.model, getattr(self, '_roll', (0, 0))
        out, ptrs, dev = self._outputs(out, [(n, T, m.nsensordata)] * 2, [np.float32] * 2)
        self._check(self._lib.fb_rollout_sensor_read(self._h, *ptrs, int(dev)), 'fb_rollout_sensor_read')
        return tuple(out)

    # ---- the iLQR backward pass (fb_lqr*; flybody_b200.trajopt is the front end)
    def lqr(self, A, B, q, r, Q, R, Qf, mu, lower=None, upper=None):
        """the Riccati backward pass of L problems: A [L, T, nx, nx], B [L, T, nx, nu] (fp32), q [L, T + 1, nx], r [L, T, nu], the
        diagonal weights Q [nx], R [nu], Qf [nx] and mu [L] (fp64), host arrays (see the header); read with lqr_read().  With bounds
        lower and / or upper [L, T, nu] (fp64, the other one -inf / +inf when None) on du = u - ubar it is the box-DDP pass
        (fb_lqr_box), whose clamped sets and QP records lqr_box_read() returns."""
        m = self.model
        nx, nu = 2 * m.nv + m.na, m.nu
        L, T = np.shape(A)[:2]
        want = [('A', (L, T, nx, nx), np.float32), ('B', (L, T, nx, nu), np.float32), ('q', (L, T + 1, nx), np.float64),
                ('r', (L, T, nu), np.float64), ('Q', (nx,), np.float64), ('R', (nu,), np.float64), ('Qf', (nx,), np.float64),
                ('mu', (L,), np.float64)]
        args = [A, B, q, r, Q, R, Qf, mu]
        box = lower is not None or upper is not None
        if box:
            want += [('lower', (L, T, nu), np.float64), ('upper', (L, T, nu), np.float64)]
            args += [np.full((L, T, nu), -np.inf) if lower is None else lower, np.full((L, T, nu), np.inf) if upper is None else upper]
        keep = [np.ascontiguousarray(x, dt) for x, (_, _, dt) in zip(args, want)]
        for x, (name, shape, _) in zip(keep, want):
            if x.shape != shape:
                raise ValueError(f'{name} {x.shape} against {shape}')
        fn = 'fb_lqr_box' if box else 'fb_lqr'
        self._check(getattr(self._lib, fn)(self._h, int(L), int(T), *[x.ctypes.data for x in keep], 0), fn)
        self._lqr = (int(L), int(T))

    def lqr_box_read(self):
        """-> (clamped [L, T, nu] (-1 at lower, +1 at upper, 0 free), qp [L, T, 2] (accepted Newton steps, stop reason)) int32 of the
        last lqr with bounds"""
        L, T = getattr(self, '_lqr', (0, 0))
        out = [np.zeros((L, T, self.model.nu), np.int32), np.zeros((L, T, 2), np.int32)]
        self._check(self._lib.fb_lqr_box_read(self._h, *[x.ctypes.data for x in out], 0), 'fb_lqr_box_read')
        return tuple(out)

    def lqr_read(self):
        """-> (K [L, T, nu, nx], k [L, T, nu], dV [L, 2] fp64, status [L] int32) of the last lqr"""
        m, (L, T) = self.model, getattr(self, '_lqr', (0, 0))
        out = [np.zeros((L, T, m.nu, 2 * m.nv + m.na)), np.zeros((L, T, m.nu)), np.zeros((L, 2)), np.zeros(L, np.int32)]
        self._check(self._lib.fb_lqr_read(self._h, *[x.ctypes.data for x in out], 0), 'fb_lqr_read')
        return tuple(out)

    # ---- sampling-based MPC (fb_plan*; flybody_b200.trajopt.sample_plan / mpc are the front ends)
    def plan_program(self, n_samples=0, sigma=None, Q=None, R=None, Qf=None, temperature=0.0, hold=1):
        """the program of the plans that follow: n_samples samples per problem, noise scale sigma [nu], diagonal weights Q [nx], R [nu],
        Qf [nx] (Q when None), temperature (> 0: MPPI, 0: predictive sampling) and hold control steps per noise knot; n_samples = 0
        clears it (see the header)"""
        m = self.model
        if not n_samples:
            self._check(self._lib.fb_plan_program(self._h, None), 'fb_plan_program')
            return
        nx = 2 * m.nv + m.na
        Qf = Q if Qf is None else Qf
        keep = [np.ascontiguousarray(np.broadcast_to(np.asarray(x, dt), (n,))) for x, dt, n in
                ((sigma, np.float32, m.nu), (Q, np.float64, nx), (R, np.float64, m.nu), (Qf, np.float64, nx))]
        f64 = C.POINTER(C.c_double)
        prog = FbPlanProgram(n_samples=int(n_samples), hold=int(hold), temperature=float(temperature),
                           sigma=keep[0].ctypes.data_as(C.POINTER(C.c_float)), Q=keep[1].ctypes.data_as(f64),
                           R=keep[2].ctypes.data_as(f64), Qf=keep[3].ctypes.data_as(f64))
        self._check(self._lib.fb_plan_program(self._h, C.byref(prog)), 'fb_plan_program')
        self._plan_k = int(n_samples)

    def plan(self, slots, mean, x_ref, seeds, u_ref=None, n_substeps=1, n_iter=1, T=None, is_device=False):
        """n_iter iterations of the program's planner for L problems: problem l from bank row slots[l] with seed seeds[l] (host ints),
        mean [L, T, nu], x_ref [L, T + 1, nq + nv + na], u_ref [L, T, nu] (None: 0) (host arrays, or device pointers / CUDA tensors'
        data_ptr() with is_device=True and T given).  The envs' states are a workspace afterwards.  Read the results with plan_read()."""
        m = self.model
        s = np.ascontiguousarray(np.asarray(slots).reshape(-1), np.int32)
        L = len(s)
        sd = np.ascontiguousarray(np.asarray(seeds, np.int64).reshape(-1) & 0xffffffff, np.uint32)
        if len(sd) != L:
            raise ValueError(f'{len(sd)} seeds for {L} problems')
        T = int(T if is_device else np.shape(mean)[1])
        ptrs, _keep = self._inputs([('mean', mean, (L, T, m.nu)), ('x_ref', x_ref, (L, T + 1, m.nq + m.nv + m.na)),
                                    ('u_ref', u_ref, (L, T, m.nu))], is_device)
        self._check(self._lib.fb_plan(self._h, s.ctypes.data, L, T, int(n_substeps), int(n_iter), sd.ctypes.data, *ptrs,
                                      int(bool(is_device))), 'fb_plan')
        self._plan = (L, T, int(n_iter), getattr(self, '_plan_k', 0))

    def plan_read(self, out=None, samples=True):
        """-> (mean [L, T, nu] f32, cost [L, n_iter, 2] f64 (the nominal's and the best cost of each iteration), sample_cost [L, K] f64
        and samples [L, K, T, nu] f32 of the last iteration, status [L] i32) of the last plan; samples=False leaves sample_cost and
        samples on the device (None); out: the five arrays to fill instead (numpy arrays, or torch tensors, CUDA ones by device pointer;
        None: not read)"""
        m, (L, T, n_iter, K) = self.model, getattr(self, '_plan', (0, 0, 0, 0))
        shapes = [(L, T, m.nu), (L, n_iter, 2), (L, K), (L, K, T, m.nu), (L,)]
        dtypes = [np.float32, np.float64, np.float64, np.float32, np.int32]
        if out is None and not samples:
            out = [np.zeros(sh, dt) if i in (0, 1, 4) else None for i, (sh, dt) in enumerate(zip(shapes, dtypes))]
        out, ptrs, dev = self._outputs(out, shapes, dtypes)
        self._check(self._lib.fb_plan_read(self._h, *ptrs, int(dev)), 'fb_plan_read')
        return tuple(out)

    # ---- system identification (fb_sid_*; flybody_b200.sysid is the front end)
    def sid_accumulate(self, query, L, problem, weight, target=None, sample_weight=None, reset=True, is_device=False):
        """add the weighted normal equations of the last fd_param_transition (query SID_TRANSITION; target: x'_obs [n, nq + nv + na],
        weight [nx]) or fd_param_inverse (SID_INVERSE; target: the qfrc_inverse target [n, nv], None: 0; weight [nv]) to L fit problems:
        FD problem i goes to fit problem problem[i] (host ints, -1: skipped), with sample_weight [n] (None: 1).  target and sample_weight
        are host arrays, or device pointers / CUDA tensors' data_ptr() with is_device=True; weight is a host array (fp64).  reset starts
        the L problems' sums from 0, else the call adds to them (see the header).  Read the sums with sid_read()."""
        m = self.model
        inv = query == SID_INVERSE
        pb = np.ascontiguousarray(np.asarray(problem).reshape(-1), np.int32)
        n = len(pb)
        rows, nr = (m.nv, m.nv) if inv else (2 * m.nv + m.na, m.nq + m.nv + m.na)
        w = np.ascontiguousarray(np.broadcast_to(np.asarray(weight, np.float64), (rows,)))
        ptrs, _keep = self._inputs([('target', target, (n, nr)), ('sample_weight', sample_weight, (n,))], is_device)
        self._check(self._lib.fb_sid_accumulate(self._h, int(query), int(L), pb.ctypes.data, n, ptrs[0], w.ctypes.data, ptrs[1],
                                                int(bool(reset)), int(bool(is_device))), 'fb_sid_accumulate')
        self._sid = (int(L), (getattr(self, '_fdpi_n', (0, 0)) if inv else getattr(self, '_fdp_n', (0, 0)))[1])

    def sid_read(self, out=None):
        """-> (H [L, k, k], g [L, k], cost [L] f64, count [L], bad [L] i32) of the sums; out: the five arrays to fill instead (numpy
        arrays, or torch tensors, CUDA ones by device pointer; None: not read)"""
        L, k = getattr(self, '_sid', (0, 0))
        out, ptrs, dev = self._outputs(out, [(L, k, k), (L, k), (L,), (L,), (L,)], [np.float64] * 3 + [np.int32] * 2)
        self._check(self._lib.fb_sid_read(self._h, *ptrs, int(dev)), 'fb_sid_read')
        return tuple(out)

    def reset(self, qpos=None, qvel=None, env_ids=None):
        n = self.n_envs if env_ids is None else len(env_ids)
        ids = None if env_ids is None else np.ascontiguousarray(env_ids, np.int32)
        qp = None if qpos is None else np.ascontiguousarray(np.broadcast_to(np.asarray(qpos, np.float32), (n, self.model.nq)))
        qv = None if qvel is None else np.ascontiguousarray(np.broadcast_to(np.asarray(qvel, np.float32), (n, self.model.nv)))
        self._check(self._lib.fb_reset(self._h, None if ids is None else ids.ctypes.data, n,
                                       None if qp is None else qp.ctypes.data, None if qv is None else qv.ctypes.data), 'fb_reset')

    def reset_hold(self, env_ids, qpos, qvel=None):
        ids = np.ascontiguousarray(env_ids, np.int32)
        qp = np.ascontiguousarray(np.broadcast_to(np.asarray(qpos, np.float32), (len(ids), self.model.nq)))
        qv = None if qvel is None else np.ascontiguousarray(np.broadcast_to(np.asarray(qvel, np.float32), (len(ids), self.model.nv)))
        self._check(self._lib.fb_reset_hold(self._h, ids.ctypes.data, len(ids), qp.ctypes.data,
                                            None if qv is None else qv.ctypes.data), 'fb_reset_hold')

    def set_action_map(self, ctrl_index):
        """fb_set_action_map: afterwards set_control takes rows in action order (see the header)."""
        if ctrl_index is None:
            self._n_ctrl_cols = self.model.nu
            self._check(self._lib.fb_set_action_map(self._h, None, 0), 'fb_set_action_map')
            return
        idx = np.ascontiguousarray(ctrl_index, np.int32)
        self._check(self._lib.fb_set_action_map(self._h, idx.ctypes.data, len(idx)), 'fb_set_action_map')
        self._n_ctrl_cols = len(idx)

    def step(self, n_substeps):
        self._check(self._lib.fb_step(self._h, int(n_substeps)), 'fb_step')

    def forward(self):
        self._check(self._lib.fb_forward(self._h), 'fb_forward')

    def sync(self):
        self._check(self._lib.fb_sync(self._h), 'fb_sync')

    def set_solver(self, tolerance=0.0, max_iter=0):
        self._lib.fb_set_solver(self._h, float(tolerance), int(max_iter))

    @property
    def launch_count(self):
        return int(self._lib.fb_launch_count(self._h))

    @property
    def last_step_ms(self):
        return float(self._lib.fb_last_step_ms(self._h))

    @property
    def stream(self):
        return self._lib.fb_stream(self._h)

    def obs_ptr(self):
        p = C.c_void_p()
        n = C.c_int()
        self._check(self._lib.fb_obs_ptr(self._h, C.byref(p), C.byref(n)), 'fb_obs_ptr')
        return p.value, n.value

    def obs_program(self, items, lists, root_body, n_sub, ref_qpos=None):
        """items: [(kind, a, b)], lists: flat int list referenced by QPOS/QVEL/SITES items. Returns row length."""
        kind = np.ascontiguousarray([i[0] for i in items], np.int32)
        a = np.ascontiguousarray([i[1] for i in items], np.int32)
        b = np.ascontiguousarray([i[2] for i in items], np.int32)
        lst = np.ascontiguousarray(lists if len(lists) else [0], np.int32)
        ref = None if ref_qpos is None else np.ascontiguousarray(ref_qpos, np.float32)
        p = FbObsProgram(len(items), kind.ctypes.data_as(C.POINTER(C.c_int32)), a.ctypes.data_as(C.POINTER(C.c_int32)),
                         b.ctypes.data_as(C.POINTER(C.c_int32)), len(lists), lst.ctypes.data_as(C.POINTER(C.c_int32)),
                         int(root_body), int(n_sub), 0 if ref is None else ref.shape[0],
                         None if ref is None else ref.ctypes.data_as(C.POINTER(C.c_float)))
        dim = self._lib.fb_obs_program(self._h, C.byref(p))
        if dim < 0:
            raise StepperError(f'fb_obs_program failed ({dim}): {self._lib.fb_last_error(self._h).decode()}')
        self._tobs_dim = dim
        return dim

    def ref_slots(self, slot_len):
        """one reference table [slot_len][7] per env instead of the shared one (fb_ref_slots)."""
        self._check(self._lib.fb_ref_slots(self._h, int(slot_len)), 'fb_ref_slots')
        self._slot_len = int(slot_len)

    def ref_slot_write(self, env_ids, rows):
        ids = np.ascontiguousarray(env_ids, np.int32)
        r = np.ascontiguousarray(rows, np.float32)
        assert r.shape == (len(ids), self._slot_len, 7), r.shape
        self._check(self._lib.fb_ref_slot_write(self._h, ids.ctypes.data, len(ids), r.ctypes.data), 'fb_ref_slot_write')

    # ---- device-side task logic (fb_task_*)
    def task_program(self, **kw):
        """upload an FbTaskProgram; array arguments are numpy arrays (kept alive for the duration of the call)."""
        keep = []

        def fp(a):
            a = np.ascontiguousarray(a, np.float32); keep.append(a)
            return a.ctypes.data_as(C.POINTER(C.c_float))

        def ip(a):
            a = np.ascontiguousarray(a, np.int32); keep.append(a)
            return a.ctypes.data_as(C.POINTER(C.c_int32))
        p = FbTaskProgram()
        for name, ctype in FbTaskProgram._fields_:
            if name not in kw or kw[name] is None:
                continue
            v = kw[name]
            if ctype is C.POINTER(C.c_float):
                v = fp(v)
            elif ctype is C.POINTER(C.c_int32):
                v = ip(v)
            elif ctype in (C.c_float * 2, C.c_float * 3, C.c_float * 4):
                v = ctype(*[float(x) for x in v])
            setattr(p, name, v)
        self._check(self._lib.fb_task_program(self._h, C.byref(p)), 'fb_task_program')

    def task_step(self, action, n_substeps, is_device=False):
        if is_device:
            self._check(self._lib.fb_task_step(self._h, C.c_void_p(int(action)), 1, int(n_substeps)), 'fb_task_step')
        else:
            a = np.ascontiguousarray(action, np.float32)
            self._keep_action = a                  # the copy is asynchronous
            self._check(self._lib.fb_task_step(self._h, a.ctypes.data, 0, int(n_substeps)), 'fb_task_step')

    def task_reset_all(self):
        self._check(self._lib.fb_task_reset_all(self._h), 'fb_task_reset_all')

    def task_request_reset(self, env_ids):
        ids = np.ascontiguousarray(env_ids, np.int32)
        self._check(self._lib.fb_task_request_reset(self._h, ids.ctypes.data, len(ids)), 'fb_task_request_reset')

    def task_uniform_rows(self, env_ids, rows):
        ids = np.ascontiguousarray(env_ids, np.int32); u = np.ascontiguousarray(rows, np.float32).reshape(len(ids), 8)
        self._check(self._lib.fb_task_uniform_rows(self._h, ids.ctypes.data, len(ids), u.ctypes.data), 'fb_task_uniform_rows')

    def hfield_bank(self, heights):
        h = np.ascontiguousarray(heights, np.float32).reshape(len(heights), -1)
        assert h.shape[1] == self._hfield_cells, (h.shape, self._hfield_cells)
        self._check(self._lib.fb_hfield_bank(self._h, h.shape[0], h.ctypes.data), 'fb_hfield_bank')

    def ref_bank(self, traj_len, rows):
        """fb_ref_bank: flight trajectories as rows [sum(traj_len)][15] (root qpos 7, CoM qvel 6, CoM x, y 2), one after the other."""
        ln = np.ascontiguousarray(traj_len, np.int32)
        r = np.ascontiguousarray(rows, np.float32)
        assert r.shape == (int(ln.sum()), 15), (r.shape, int(ln.sum()))
        self._check(self._lib.fb_ref_bank(self._h, len(ln), ln.ctypes.data, r.ctypes.data), 'fb_ref_bank')

    def ref_bank_wide(self, traj_len, rows):
        """fb_ref_bank_wide: trajectories as rows [sum(traj_len)][w >= 15], one after the other; the first 15 columns as for ref_bank
        (walking: root qpos 7, root qvel 6, root x, y 2), then the task's own columns (walking: the reward features)."""
        ln = np.ascontiguousarray(traj_len, np.int32)
        r = np.ascontiguousarray(rows, np.float32)
        assert r.ndim == 2 and r.shape[0] == int(ln.sum()) and r.shape[1] >= 15, (r.shape, int(ln.sum()))
        self._check(self._lib.fb_ref_bank_wide(self._h, len(ln), ln.ctypes.data, r.shape[1], r.ctypes.data), 'fb_ref_bank_wide')

    def task_ref_pick(self, env_ids, traj, start):
        """pin the trajectory and start step of the listed envs' next reset (fb_task_ref_pick)"""
        ids = np.ascontiguousarray(env_ids, np.int32)
        tr, s0 = np.ascontiguousarray(traj, np.int32), np.ascontiguousarray(start, np.int32)
        assert tr.shape == s0.shape == ids.shape, (ids.shape, tr.shape, s0.shape)
        self._check(self._lib.fb_task_ref_pick(self._h, ids.ctypes.data, len(ids), tr.ctypes.data, s0.ctypes.data), 'fb_task_ref_pick')

    def task_ref_state(self):
        """-> (trajectory, start step) int32 [n_envs] of every env's running episode (fb_task_ref_state)"""
        traj, start = np.zeros(self.n_envs, np.int32), np.zeros(self.n_envs, np.int32)
        self._check(self._lib.fb_task_ref_state(self._h, traj.ctypes.data, start.ctypes.data), 'fb_task_ref_state')
        return traj, start

    def task_set_reset_noise(self, amp):
        self._check(self._lib.fb_task_set_reset_noise(self._h, float(amp)), 'fb_task_set_reset_noise')

    def task_episodes(self):
        out = np.zeros(self.n_envs, np.int32)
        self._check(self._lib.fb_task_episodes(self._h, out.ctypes.data), 'fb_task_episodes')
        return out

    def task_uniforms(self, env_ids, u):
        ids = np.ascontiguousarray(env_ids, np.int32); uu = np.ascontiguousarray(u, np.float32)
        self._check(self._lib.fb_task_uniforms(self._h, ids.ctypes.data, len(ids), uu.ctypes.data), 'fb_task_uniforms')

    def task_ptrs(self):
        o, n, r = C.c_void_p(), C.c_int(), C.c_void_p()
        self._check(self._lib.fb_task_ptrs(self._h, C.byref(o), C.byref(n), C.byref(r)), 'fb_task_ptrs')
        return o.value, n.value, r.value

    def task_read(self, obs_out, out4):
        self._check(self._lib.fb_task_read(self._h, obs_out.ctypes.data, out4.ctypes.data), 'fb_task_read')

    # ---- eye cameras (fb_eye_program / fb_render_eyes)
    def eye_program(self, bodies, pos, quat, fovy_deg=150.0, size=32, nrow=0, ncol=0, half_size=20.0, z_offset=0.0, zfar=50.0,
                    sky_top=(0.33, 0.47, 0.70), sky_horizon=(0.50, 0.56, 0.65), ground=(0.15, 0.11, 0.08), ambient=0.4, diffuse=0.8):
        """The default palette is calibrated, not copied: MuJoCo's GL image cannot be reproduced, but the gray-level statistics the
        reference's vision network assumes can -- `VisNet` normalises with mean 77 / std 56 "from the trench task"
        (network_factory_vis.py:158-162); with these colours the eyes of `vision_guided_flight('trench')` measure 76 / 56 (bumps: 80 / 57),
        tests/test_eyes.py::test_eye_statistics_match_the_vision_network_normalisation."""
        p = FbEyeProgram()
        p.n_cam = len(bodies)
        for c in range(p.n_cam):
            p.body[c] = int(bodies[c])
            for k in range(3):
                p.pos[c][k] = float(pos[c][k])
            for k in range(4):
                p.quat[c][k] = float(quat[c][k])
        p.fovy_deg, p.size, p.nrow, p.ncol, p.half_size, p.z_offset, p.zfar = fovy_deg, size, nrow, ncol, half_size, z_offset, zfar
        for k in range(3):
            p.sky_top[k], p.sky_horizon[k], p.ground[k] = sky_top[k], sky_horizon[k], ground[k]
        p.ambient, p.diffuse = ambient, diffuse
        self._check(self._lib.fb_eye_program(self._h, C.byref(p)), 'fb_eye_program')
        self._eye_shape = (self.n_envs, p.n_cam, size, size, 3)
        self._hfield_cells = nrow * ncol

    def hfield_collision(self, geom, size, nrow, ncol, pair_geom):
        """turn on the heightfield narrowphase for the model's terrain geom (fb_hfield_collision)."""
        sz = np.ascontiguousarray(size, np.float32); pg = np.ascontiguousarray(pair_geom, np.int32)
        self._check(self._lib.fb_hfield_collision(self._h, int(geom), sz.ctypes.data, int(nrow), int(ncol), pg.ctypes.data, len(pg)), 'fb_hfield_collision')
        self._hfield_cells = int(nrow) * int(ncol)

    def hfield_write(self, env_ids, heights):
        ids = np.ascontiguousarray(env_ids, np.int32)
        h = np.ascontiguousarray(heights, np.float32).reshape(len(ids), -1)
        assert h.shape[1] == self._hfield_cells, (h.shape, self._hfield_cells)
        self._check(self._lib.fb_hfield_write(self._h, ids.ctypes.data, len(ids), h.ctypes.data), 'fb_hfield_write')

    def eyes_ptr(self):
        """(device pointer, bytes per env) of the eye-camera images (valid from eye_program until the next eye_program or close;
        rewritten by every render_eyes)"""
        p, n = C.c_void_p(), C.c_int()
        self._check(self._lib.fb_eyes_ptr(self._h, C.byref(p), C.byref(n)), 'fb_eyes_ptr')
        return p.value, n.value

    def render_eyes_async(self):
        """launch the eye renderer on the stepper's stream; the images stay on the device (eyes_ptr)"""
        self._check(self._lib.fb_render_eyes(self._h), 'fb_render_eyes')

    def render_eyes(self, out=None):
        """-> uint8 [n_envs, n_cam, size, size, 3] rendered from the current body poses."""
        self._check(self._lib.fb_render_eyes(self._h), 'fb_render_eyes')
        out = np.empty(self._eye_shape, np.uint8) if out is None else out
        self._check(self._lib.fb_eyes_read(self._h, out.ctypes.data), 'fb_eyes_read')
        return out

    def task_inputs(self, step_idx, first):
        si = np.ascontiguousarray(step_idx, np.int32)
        fi = np.ascontiguousarray(first, np.uint8)
        self._check(self._lib.fb_task_inputs(self._h, si.ctypes.data, fi.ctypes.data), 'fb_task_inputs')

    def read_task_obs(self, out):
        self._check(self._lib.fb_pack_obs(self._h), 'fb_pack_obs')
        self._check(self._lib.fb_read_task_obs(self._h, out.ctypes.data), 'fb_read_task_obs')
        return out

    def profile(self, enable=True):
        self._lib.fb_profile(self._h, 1 if enable else 0)

    def profile_read(self):
        ms = np.zeros(16, np.float64)
        cnt = np.zeros(16, np.int64)
        n = self._lib.fb_profile_read(self._h, ms.ctypes.data, cnt.ctypes.data, 16)
        return {self._lib.fb_profile_name(k).decode(): (float(ms[k]), int(cnt[k])) for k in range(n)}

    def step_kernel_smem(self):
        """{stage name: (dynamic shared bytes per CTA as launched, resident CTAs per SM at that size)} of the seven step
        kernels (fb_step_kernel_smem; the CTA count is 0 in a build without a device)."""
        out, nb, blocks = {}, C.c_int(), C.c_int()
        for k in range(16):
            rc = self._lib.fb_step_kernel_smem(self._h, k, C.byref(nb), C.byref(blocks))
            if rc == 0:
                out[self._lib.fb_profile_name(k).decode()] = (nb.value, blocks.value)
            elif rc != -1:
                self._check(rc, 'fb_step_kernel_smem')
        return out

    def set_control_device(self, dev_ptr):
        """ctrl already resident on the device as contiguous rows [n_envs][nu] fp32."""
        self._check(self._lib.fb_set_ctrl(self._h, C.c_void_p(dev_ptr), 1), 'fb_set_ctrl')

    def pack_obs(self):
        self._check(self._lib.fb_pack_obs(self._h), 'fb_pack_obs')

    @property
    def record_bytes(self):
        """bytes of device state per env (one record: persistent state + per-substep intermediates)."""
        return 4 * int(self._lib.fb_record_stride(self._h))

    @property
    def n_envs_padded(self):
        return int(self._lib.fb_n_envs_padded(self._h))

    def read_obs(self, out=None):
        """Pack + copy the per-env observation record [N, obs_dim] (see fb_pack_obs in the header)."""
        _, dim = self.obs_ptr()
        if out is None:
            out = np.empty((self.n_envs, dim), np.float32)
        self._check(self._lib.fb_pack_obs(self._h), 'fb_pack_obs')
        self._check(self._lib.fb_read_obs(self._h, out.ctypes.data), 'fb_read_obs')
        return out

    def obs_layout(self):
        m = self.model
        off, lay = 0, {}
        for name, n in (('qpos', m.nq), ('qvel', m.nv), ('act', m.na), ('sensor_mean', m.nsensordata),
                        ('sensordata', m.nsensordata), ('root_xpos', 3), ('root_xmat', 9),
                        ('site_xpos', 3 * m.nsite), ('flags', 1), ('qacc_sq', 1), ('time', 1)):
            lay[name] = slice(off, off + n)
            off += n
        return lay

    def version(self):
        return self._lib.fb_version().decode()
