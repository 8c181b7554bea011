"""Drop-in, batched counterparts of the reference's environment factories
(`flybody/fly_envs.py:100-155` walk_imitation, `:30-97` flight_imitation).

`walk_imitation(n_envs=N)` returns a `WalkImitationEnv` (a `BatchedFlyEnv`) with the `dm_env` surface of the reference
(`reset()`, `step(action)`, `action_spec()`, `observation_spec()`, `control_timestep()`,
`physics.timestep()`, `task._traj_generator.set_next_trajectory`) where every array carries a
leading batch dimension N.  With `n_envs=None` a single environment without the batch dimension
is returned (what the reference's tests construct).  The physics is the CUDA stepper; the task
logic mirrors `flybody/tasks/walk_imitation.py` / `tasks/base.py` in vectorised numpy.

One class per task: `_TaskEnv` is the episode shell (host and device) of every env, `BatchedFlyEnv` adds the FruitFly walker, and
`TemplateTaskEnv`, `WalkOnBallEnv`, `WalkImitationEnv` and `FlightImitationEnv` (the last two over `_ImitationEnv`: ghost and reference)
are its tasks; `vision_env.BatchedVisionFlightEnv` is a `_TaskEnv` of its own.
"""
import collections
import hashlib
import types

import numpy as np

from . import rewards as rw
from . import stepper as st
from .dm_env_shim import Array, BoundedArray, StepType, TimeStep
from .flymodel import load_model

from .synthetic import (_WALK_CONTROL_TIMESTEP, _WALK_PHYSICS_TIMESTEP, _TERMINAL_LINVEL, _TERMINAL_ANGVEL,  # noqa: F401
                        _FLY_CONTROL_TIMESTEP, _FLY_PHYSICS_TIMESTEP, _TERMINAL_HEIGHT, _TERMINAL_QACC, _ACTION_CLASS_ORDER,
                        mult_quat, reciprocal_quat, quat_dist_short_arc, linear_tolerance, constant_speed_trajectory,
                        rotate_vec_with_quat, com2root, root2com, _COM_OFFSET)
from .trajectory_loaders import (HDF5FlightTrajectoryLoader, HDF5WalkingTrajectoryLoader,  # noqa: F401
                                 InferenceFlightTrajectoryLoader, InferenceWalkingTrajectoryLoader)


class BatchedWingBeatPatternGenerator:
    """Vectorised `WingBeatPatternGenerator` (reference `tasks/pattern_generators.py:8-203`): per-env phase-preserving
    frequency modulation of one wing-beat cycle.  Tables are built once (one resampled, repeated cycle per discrete beat
    frequency, padded to a common length); the per-env state is (filtered frequency, table index, position in table)."""

    def __init__(self, n_envs, base_pattern_path=None, base_beat_freq=218.0, rel_freq_range=0.05, num_freqs=201,
                 min_repeats=10, max_repeats=20, dt_ctrl=_FLY_CONTROL_TIMESTEP, ctrl_filter=0.5 / 218.0):
        if base_pattern_path is None:       # the reference's synthetic stand-in cycle (pattern_generators.py:53-59)
            x = np.linspace(0, 2 * np.pi, 500)
            cycle = np.stack([1.1 * np.sin(x - np.pi / 2) + 0.3, 0.25 * np.sin(1.5 * x) - 0.1, 1.35 * np.sin(x) + 0.8], 1)
        else:
            cycle = np.load(base_pattern_path)
        cycle = np.concatenate([cycle, cycle], 1)              # both wings
        n_pts = cycle.shape[0]
        self.base_beat_freq, self.rel_freq_range, self.ctrl_filter, self._dt = base_beat_freq, rel_freq_range, ctrl_filter, dt_ctrl
        self._rate = np.exp(-dt_ctrl / ctrl_filter) if ctrl_filter != 0.0 else 0.0
        self.beat_freqs = np.linspace((1 - rel_freq_range) * base_beat_freq, (1 + rel_freq_range) * base_beat_freq, num_freqs)
        trajs, phases = [], []
        reps = np.arange(min_repeats, max_repeats + 1)
        for f in self.beat_freqs:
            period = 1.0 / f
            err = ((reps * period) % dt_ctrl) / dt_ctrl        # mismatch of the seam, in control steps
            i_over, i_under = int(np.argmin(err)), int(np.argmin(np.abs(1 - err)))
            if err[i_over] < abs(1 - err[i_under]):
                pick, shift = i_over, dt_ctrl
            else:
                pick, shift = i_under, 0.0
            n_rep = pick + 1                                    # (sic) the reference repeats argmin+1 cycles
            data = np.tile(cycle, (n_rep, 1))
            ph = np.linspace(0, n_rep, n_rep * n_pts, endpoint=False)
            total = data.shape[0] * (period / n_pts)
            t_data = np.linspace(0, total, data.shape[0])
            t_ctrl = np.arange(0, total - shift, dt_ctrl)
            trajs.append(np.stack([np.interp(t_ctrl, t_data, data[:, k]) for k in range(data.shape[1])], 1))
            phases.append(np.interp(t_ctrl, t_data, ph))
        self.lengths = np.array([t.shape[0] for t in trajs])
        L = int(self.lengths.max())
        self.traj = np.zeros((num_freqs, L, cycle.shape[1]))
        self.phase = np.full((num_freqs, L), np.inf)            # padding never wins an argmin
        for i, (t, ph) in enumerate(zip(trajs, phases)):
            self.traj[i, :t.shape[0]] = t
            self.phase[i, :t.shape[0]] = ph
        self.phase_mod = np.where(np.isfinite(self.phase), np.mod(self.phase, 1.0, where=np.isfinite(self.phase), out=np.zeros_like(self.phase)), np.inf)
        self.freq = np.full(n_envs, base_beat_freq)
        self.idx = np.zeros(n_envs, np.int64)
        self.pos = np.zeros(n_envs, np.int64)

    def _nearest(self, freq):
        return np.abs(self.beat_freqs[None, :] - np.asarray(freq)[:, None]).argmin(1)

    def reset(self, ids, initial_phase):
        """-> (wing qpos [n, 6], wing qvel [n, 6]) at the requested phase of the base frequency."""
        ids = np.asarray(ids)
        self.freq[ids] = self.base_beat_freq
        idx = self._nearest(self.freq[ids])
        pos = np.abs(np.asarray(initial_phase)[:, None] - self.phase[idx]).argmin(1)
        self.idx[ids], self.pos[ids] = idx, pos
        nxt = np.minimum(pos + 1, self.lengths[idx] - 1)
        q = self.traj[idx, pos]
        return q, (self.traj[idx, nxt] - q) / self._dt

    def step(self, ctrl_freq, active=None):
        """advance every (active) env by one control step at its requested beat frequency -> wing angles [N, 6]."""
        act = np.ones(self.freq.shape[0], bool) if active is None else np.asarray(active, bool)
        pos = np.where(act, (self.pos + 1) % self.lengths[self.idx], self.pos)
        freq = ctrl_freq if self.ctrl_filter == 0.0 else self.freq * self._rate + ctrl_freq * (1 - self._rate)
        self.freq = np.where(act, freq, self.freq)
        new = self._nearest(self.freq)
        sw = np.nonzero(act & (new != self.idx))[0]
        if sw.size:                                              # keep the phase within the beat when changing table
            cur = self.phase_mod[self.idx[sw], pos[sw]]
            pos[sw] = np.abs(cur[:, None] - self.phase_mod[new[sw]]).argmin(1)
            self.idx[sw] = new[sw]
        self.pos = pos
        return self.traj[self.idx, self.pos]



_WALK_REWARD_WEIGHTS = (20, 1, 1, 1)            # DeepMimic factor weights of walk_imitation (walk_imitation.py:152-177)
_WING_RETRACT_MARGIN = 3.0                      # ... and the margin of its wing-retraction factors


class _FeatureBank:
    """Full-body reference features of the walking snippets in use, concatenated row-wise (append-only, cached by
    trajectory index) so that the per-env reward gathers are single fancy-index reads."""

    def __init__(self):
        self._off, self._n = {}, 0
        self.qpos = self.qvel = self.root2site = self.joint_quat = None

    @staticmethod
    def _append(buf, n_used, new):
        new = np.asarray(new, np.float64)
        if buf is None:
            buf = np.zeros((max(4 * new.shape[0], 1024),) + new.shape[1:])
        while n_used + new.shape[0] > buf.shape[0]:
            buf = np.concatenate([buf, np.zeros_like(buf)], 0)
        buf[n_used:n_used + new.shape[0]] = new
        return buf

    def offset_of(self, idx, snip):
        key = None if idx is None else int(idx)
        if key is not None and key in self._off:
            return self._off[key]
        T = snip['qpos'].shape[0]
        self.qpos = self._append(self.qpos, self._n, snip['qpos'])
        self.qvel = self._append(self.qvel, self._n, snip['qvel'])
        self.root2site = self._append(self.root2site, self._n, snip['root2site'])
        self.joint_quat = self._append(self.joint_quat, self._n, snip['joint_quat'])
        off = self._n
        self._n += T
        if key is not None:
            self._off[key] = off
        return off


class _PhysicsFacade:
    """The slice of `dm_control.mjcf.Physics` the reference's callers touch (SURVEY.md 8(b))."""

    def __init__(self, env):
        self._env = env

    def timestep(self):
        return self._env._physics_timestep

    def time(self):
        return self._env._time.copy() if self._env._batched else float(self._env._time[0])

    @property
    def stepper(self):
        return self._env._sim


class _ImitationTask:
    """What the reference's callers reach through `env.task` (`tasks/base.py:22-268`)."""
    name = 'FruitFlyTask'

    def __init__(self, env, traj_generator, terminal_com_dist, future_steps, time_limit, control_timestep):
        self._env = env
        self._traj_generator = traj_generator
        self._terminal_com_dist = terminal_com_dist
        self._future_steps = future_steps
        self._time_limit = time_limit
        self._max_episode_steps = round(time_limit / control_timestep) + 1
        self._ghost_offset = np.zeros(3)
        self._next_traj_idx = None

    def set_next_trajectory_index(self, idx):
        self._next_traj_idx = idx


class WalkImitationTask(_ImitationTask):
    """Batched `WalkImitation` (reference `tasks/walk_imitation.py:19-203`, `tasks/base.py:367-428`)."""


class TemplateTask:
    """What the reference's callers reach through `env.task` of `template_task` (`tasks/template_task.py`)."""
    name = 'FruitFlyTask'

    def __init__(self, env, time_limit, control_timestep):
        self._env = env
        self._traj_generator = None
        self._time_limit = time_limit
        self._future_steps = 0
        self._ghost_offset = np.zeros(3)
        self._terminal_com_dist = np.inf
        self._max_episode_steps = round(time_limit / control_timestep)


class WalkOnBallTask(TemplateTask):
    """What the reference's callers reach through `env.task` of `walk_on_ball` (`tasks/walk_on_ball.py`)."""


class FlightImitationTask(_ImitationTask):
    """Batched `FlightImitationWBPG` (reference `tasks/flight_imitation.py:16-212`, `tasks/base.py:271-364`)."""

    @property
    def _wbpg(self):
        return self._env._wbpg


# cameras `eye_right` / `eye_left` on the head (reference fruitfly.xml:335-336; the head body keeps its XML frame)
_EYE_CAMERAS = (('walker/right_eye', (0.0219, 0.0131, 0.0), (0.474, 0.688, -0.344, -0.429)),
                ('walker/left_eye', (-0.0219, 0.0131, 0.0), (0.474, 0.688, 0.344, 0.429)))
_WING_JOINTS = tuple(f'walker/wing_{a}_{s}' for s in ('left', 'right') for a in ('yaw', 'roll', 'pitch'))
# the walker's observables (dm_control lists them alphabetically; reference tests/test_core.py:9-20)
_WALKER_OBS = ('accelerometer', 'actuator_activation', 'appendages_pos', 'force', 'gyro', 'joints_pos', 'joints_vel', 'touch', 'velocimeter',
               'world_zaxis')


def _pinned(shape, dtype):
    """page-locked host buffer where torch + CUDA are present (device -> host copies at full PCIe rate), plain numpy otherwise"""
    try:
        import torch
        if torch.cuda.is_available():
            return torch.empty(shape, dtype=getattr(torch, np.dtype(dtype).name)).pin_memory().numpy()
    except Exception:
        pass
    return np.empty(shape, dtype)


def _device_tensor(ptr, shape, typestr, device):
    """zero-copy torch tensor over a buffer the library owns on `device` (typestr '<f4': fp32, '|u1': uint8)"""
    import torch
    view = types.SimpleNamespace(__cuda_array_interface__={'shape': shape, 'typestr': typestr, 'data': (int(ptr), False), 'version': 2})
    return torch.as_tensor(view, device=f'cuda:{device}')


class _TaskEnv:
    """The episode shell of every task env: N lock-stepped flies of one model on one stepper, the action layout and the dm_env specs, the
    walker's index tables and observation program, auto-reset bookkeeping, and the control step and reset -- on the host (`step`, `reset`)
    and with the task hooks on the device (`_device_step`, `step_device`).  A task states its control timestep, device task kind and
    observables as class attributes and supplies what differs through hooks: `_action` (the actions of a step), `_before_step` (the
    controls), `_after_read` (host state read off the record), `_task_after` (termination and reward), `_observation`, `_reset_envs`,
    `_ensure_programs` and the device step's `_before_device_step` / `_after_device_step`."""
    _CONTROL_TIMESTEP = _KIND = _OBS = None
    _EYE_CAMERAS = _EYE_CAMERAS                  # (the eye poses every env renders, also readable from the env)
    _N_USER = 0                 # user actions in [-1, 1] after the actuators' (flight: the beat frequency, flight_imitation.py:38)
    _HOST_CTRL = False          # the host task code builds ctrl from the actions (the wing-beat generator); else the device action map does

    def __init__(self, model, n_envs, device, lib_path, time_limit, seed, device_task):
        self._batched = n_envs is not None
        self.n_envs = N = int(n_envs) if self._batched else 1
        self.model = m = model
        self._sim = st.BatchedStepper(m, N, device=device, lib_path=lib_path)
        self._control_timestep, self._physics_timestep = self._CONTROL_TIMESTEP, float(m.opt_timestep)
        self._n_sub = int(round(self._control_timestep / self._physics_timestep))
        self._time_limit = time_limit
        self._rs = np.random.RandomState(seed)
        self._seed, self._task_kind = seed, self._KIND
        self._device_task = bool(device_task)       # task hooks evaluated on the device (fb_task_*): no host logic in step()
        # actions (reference fruitfly.py:342-379, 532-579): the actuator classes in a fixed order, then the task's user actions in
        # [-1, 1], which have no ctrl slot
        ci, idx, self._action_indices = m.meta['ctrl_indices'], [], {}
        for key in _ACTION_CLASS_ORDER:
            if ci.get(key):
                self._action_indices[key] = np.arange(len(idx), len(idx) + len(ci[key]))
                idx.extend(ci[key])
        self._ctrl_of_action, self._n_user = np.asarray(idx, np.int64), self._N_USER
        names = [m.meta['actuator_names'][i].split('/')[-1] for i in idx] + [f'user_{i}' for i in range(self._n_user)]
        rng = m.actuator_ctrlrange[idx]
        self._action_spec = BoundedArray((len(names),), np.float64, np.concatenate([rng[:, 0], -np.ones(self._n_user)]),
                                         np.concatenate([rng[:, 1], np.ones(self._n_user)]), name='\t'.join(names))
        # actions go to the device as they are where nothing rewrites them on the host: the action -> ctrl permutation and NaN -> 0 run in
        # the scatter kernel (fb_set_action_map); user actions have no ctrl slot (column -> -1, read by the device-side task code)
        self._device_action_map = not self._HOST_CTRL or self._device_task
        if self._device_action_map:
            self._sim.set_action_map(np.concatenate([self._ctrl_of_action, -np.ones(self._n_user, np.int64)]) if self._device_task
                                     else self._ctrl_of_action)
        # the walker's index tables: its free joint (-1: none, walk_on_ball's thorax is welded to the world), the observable joints, the wings
        jn, oj = m.meta['jnt_names'], m.meta['observable_joints']
        self._root_q = m.jnt_qposadr_of('walker/') if 'walker/' in jn else -1
        self._root_v = m.jnt_dofadr_of('walker/') if 'walker/' in jn else -1
        obsj = [jn.index(n) for n in oj]
        self._obs_qadr, self._obs_vadr = m.jnt_qposadr[obsj], m.jnt_dofadr[obsj]
        self._wing_qadr = np.array([m.jnt_qposadr_of(n) for n in _WING_JOINTS])
        self._wing_vadr = np.array([m.jnt_dofadr_of(n) for n in _WING_JOINTS])
        # position of the wing joints inside the joints_pos observable, where it holds them (flight, vision: the host reads wing angles there)
        self._wing_in_obs = np.array([oj.index(n) for n in _WING_JOINTS]) if _WING_JOINTS[0] in oj else None
        # per-env episode state
        self._time = np.zeros(N)
        self._needs_reset = np.ones(N, bool)
        self._step_counter = np.zeros(N, np.int64)         # control steps into the episode: the reference row the ref_* observables start at
        self._rec = None
        self._out4 = _pinned((N, 4), np.float32)
        self._dev_views = None
        self.n_resets = 0
        self.n_capacity_overflows = 0            # env-steps whose contact / constraint-row lists hit their capacity (FB_FLAGS bits 1, 2)
        self.h2d_bytes_per_step = 0
        self.d2h_bytes_per_step = 0

    # ---------------------------------------------------------------------------------- specs
    def action_spec(self):
        return self._action_spec

    def reward_spec(self):
        return Array((self.n_envs,) if self._batched else (), np.float64, name='reward')

    def discount_spec(self):
        return BoundedArray((self.n_envs,) if self._batched else (), np.float64, 0.0, 1.0, name='discount')

    def control_timestep(self):
        return self._control_timestep

    # ---------------------------------------------------------------------------------- programs
    def _upload_obs_program(self, rows, lists, shared=None):
        """Observation program: `rows` (name, width, shape, program item) in column order over the index `lists`, evaluated on the device
        (fb_obs_program; `shared`: the reference table of the ref_* items) -> the column slices and shapes by name, and the pinned record a
        step reads the rows into."""
        dim = self._sim.obs_program([r[3] for r in rows], lists, self.model.body_id('walker/thorax'), self._n_sub, shared)
        off = np.concatenate([[0], np.cumsum([r[1] for r in rows])])
        assert off[-1] == dim, (off[-1], dim)
        self._obs_slices = {r[0]: slice(int(off[i]), int(off[i + 1])) for i, r in enumerate(rows)}
        self._obs_shapes = {r[0]: r[2] for r in rows}
        self._rec = _pinned((self.n_envs, dim), np.float32)

    def _ensure_programs(self):
        """the programs are on the device (a task that uploads them in its constructor has nothing to do)"""

    def _task_program(self):
        """the fb_task_program fields every task sets; a task updates its own (ghost, thresholds, reference, wing-beat tables ...).
        Thresholds are off (+-3e38) but the bad-state |qacc|."""
        m = self.model
        sens = m.meta['sensor_names']
        return dict(kind=self._task_kind, root_qadr=self._root_q, root_vadr=self._root_v, ghost_qadr=-1, ghost_vadr=-1,
                    user_col=len(self._ctrl_of_action) if self._n_user else -1, control_timestep=self._control_timestep,
                    time_limit=self._time_limit, terminal_com_dist=3e38, terminal_linvel=3e38, terminal_angvel=3e38,
                    terminal_qacc=_TERMINAL_QACC, terminal_height=-3e38, velocimeter_adr=int(m.sensor_adr[sens.index('walker/velocimeter')]),
                    gyro_adr=int(m.sensor_adr[sens.index('walker/gyro')]), com_body=m.body_id('walker/thorax'), reset_qpos=m.qpos0,
                    n_noise=0, seed=int(self._seed) & 0xffffffff)

    def _wing_beat_program(self):
        """the fb_task_program fields of the wing-beat pattern generator `_wbpg` (flight, vision): wing joints, their ctrl columns, tables"""
        wb = self._wbpg
        return dict(n_wing=6, wing_qadr=self._wing_qadr, wing_vadr=self._wing_vadr, wing_ctrl=self._ctrl_of_action[self._action_indices['wings']],
                    n_freq=wb.traj.shape[0], tab_len=wb.traj.shape[1], wb_traj=wb.traj, wb_phase=np.where(np.isfinite(wb.phase), wb.phase, 3e38),
                    wb_phase_mod=np.where(np.isfinite(wb.phase_mod), wb.phase_mod, 3e38), wb_freqs=wb.beat_freqs, wb_len=wb.lengths,
                    wb_base_freq=wb.base_beat_freq, wb_rel_range=wb.rel_freq_range, wb_rate=wb._rate)

    def _eye_program(self, size, fovy, nrow, ncol, half_size, z_offset):
        """fb_eye_program: the two eye cameras on the head (`_EYE_CAMERAS`), rendered by the device ray caster"""
        quats = [np.asarray(q, np.float64) / np.linalg.norm(q) for _, _, q in _EYE_CAMERAS]
        head = self.model.body_id('walker/head')
        self._sim.eye_program([head, head], [p for _, p, _ in _EYE_CAMERAS], quats, fovy_deg=fovy, size=size, nrow=nrow, ncol=ncol,
                              half_size=half_size, z_offset=z_offset)
        self._eyes_dev = None           # a view of the images the program replaced, which it freed (made again by `eyes_device`)

    # -------------------------------------------------------------------------------- episode
    def request_reset(self, env_ids):
        """Restart the listed envs at the next step (their action of that step is dropped and they report FIRST), whatever their
        episode state -- an actor restarting single environments."""
        ids = np.asarray(env_ids, np.int64).reshape(-1)
        if len(ids) == 0:
            return
        if self._device_task:
            self._sim.task_request_reset(ids)
        self._needs_reset[ids] = True

    def reset(self):
        N = self.n_envs
        if self._device_task:                   # every env starts an episode in one held step (FIRST)
            self._ensure_programs()
            self._sim.task_reset_all()
            self._needs_reset[:] = True
            return self._unbatch(self._device_step(np.zeros((N, self._action_spec.shape[0]), np.float32)), first=True)
        self._reset_envs(np.arange(N))
        self._sim.task_inputs(self._step_counter, np.ones(N, np.uint8))
        obs = self._observation(self._sim.read_task_obs(self._rec))
        return self._unbatch(TimeStep(np.full(N, StepType.FIRST), np.zeros(N), np.ones(N), obs), first=True)

    def step(self, action):
        action = self._action(action)
        if self._device_task:
            return self._unbatch(self._device_step(action))
        # auto-reset of envs whose last step was LAST (composer.Environment semantics); their action is ignored
        resetting = self._needs_reset.copy()
        if resetting.any():
            self._reset_envs(np.nonzero(resetting)[0], hold=True)
        ctrl, self.h2d_bytes_per_step = self._before_step(action, resetting)
        self._sim.set_control(ctrl)
        self._step_counter += np.where(resetting, 0, 1)
        # n_sub_steps x physics.step()
        self._sim.task_inputs(self._step_counter, resetting)
        self._sim.step(self._n_sub)
        rec = self._sim.read_task_obs(self._rec)
        self.d2h_bytes_per_step = rec.nbytes
        self._time = np.where(resetting, 0.0, self._time + self._control_timestep)
        self._after_read(rec)
        obs = self._observation(rec)
        step_type, reward, discount, self._needs_reset = self._task_after(rec, obs, resetting, self._time, None)
        return self._unbatch(TimeStep(step_type, reward, discount, obs))

    def _action(self, action, host=None):
        """the actions of a step as rows [N, n_action]: an fp64 copy where the host task code rewrites them (`host`, by default where no
        device action map turns them into ctrl), else fp32 as they are"""
        host = not self._device_action_map if host is None else host
        action = (np.array(action, np.float64, copy=True) if host else np.asarray(action, np.float32)).reshape(self.n_envs, -1)
        assert action.shape[1] == self._action_spec.shape[0], f'action must have {self._action_spec.shape[0]} entries'
        return action

    def _host_ctrl(self, action):
        """ctrl [N, nu] fp32 of actions the host task code rewrote (the user actions have no ctrl slot)"""
        ctrl = np.zeros((self.n_envs, self.model.nu), np.float32)
        ctrl[:, self._ctrl_of_action] = action[:, :len(self._ctrl_of_action)]
        return ctrl

    def _after_read(self, rec):
        """host-side task state taken from the record of the step just taken"""

    def _start_episodes(self, ids, qpos, qvel, hold):
        """physics.reset() of the listed envs into (qpos, qvel) -- held through the coming step where `hold` (an auto-reset in step()) --
        and their episode counters"""
        if hold:
            self._sim.reset_hold(ids, qpos, qvel)
        else:
            self._sim.reset(qpos=qpos, qvel=qvel, env_ids=None if len(ids) == self.n_envs else ids)
        self._step_counter[ids] = 0
        self._time[ids] = 0.0
        self._needs_reset[ids] = False
        self.n_resets += len(ids)

    def _count_overflows(self, rec):
        """count the envs whose step hit a contact / constraint-row capacity (FB_FLAGS bits 1, 2: counted, not a termination)
        -> the record's _scalars columns (flags, |qacc|^2, time)"""
        scal = rec[:, self._obs_slices['_scalars']]
        self.n_capacity_overflows += int(((scal[:, 0].astype(np.int64) & 6) != 0).sum())
        return scal

    def _bad_state(self, rec):
        """non-finite / diverged state (FB_FLAGS bit 0) or |qacc| > _TERMINAL_QACC: the reference terminates on it (base.py:222-225)"""
        scal = self._count_overflows(rec)
        return ((scal[:, 0].astype(np.int64) & 1) != 0) | ~(np.sqrt(scal[:, 1].astype(np.float64)) <= _TERMINAL_QACC)

    def _end_step(self, resetting, terminate, reward, time, end_ok=None):
        """get_discount and the step type (base.py:203-225) -> step_type, reward, discount, needs_reset.  A termination costs the
        discount except where `end_ok` (walking / flight at the end of the reference); the time limit ends an episode with discount 1.
        Rows that were reset this call report FIRST (their action was ignored).  The device's tk_end_step is the same logic."""
        last = terminate | (time >= self._time_limit - 1e-9)
        discount = np.where(terminate if end_ok is None else terminate & ~end_ok, 0.0, 1.0)
        step_type = np.where(resetting, StepType.FIRST, np.where(last, StepType.LAST, StepType.MID))
        return step_type, np.where(resetting, 0.0, reward), np.where(resetting, 1.0, discount), last & ~resetting

    def _device_step(self, action):
        """one control step with the task hooks on the device: actions in, observation rows + (reward, discount, step_type) out"""
        resetting = self._needs_reset.copy()
        self._before_device_step(resetting)
        self._sim.task_step(action, self._n_sub)
        self._sim.task_read(self._rec, self._out4)
        self._count_overflows(self._rec)
        self._time = np.where(resetting, 0.0, self._time + self._control_timestep)
        self._step_counter = np.where(resetting, 0, self._step_counter + 1)
        self.n_resets += int(resetting.sum())
        self.h2d_bytes_per_step, self.d2h_bytes_per_step = action.nbytes, self._rec.nbytes + self._out4.nbytes
        self._after_device_step(resetting)
        step_type = self._out4[:, 2].astype(np.int64)
        self._needs_reset = step_type == int(StepType.LAST)
        return TimeStep(step_type, self._out4[:, 0].astype(np.float64), self._out4[:, 1].astype(np.float64), self._observation(self._rec))

    def _before_device_step(self, resetting):
        """host work before a device step; `resetting`: the envs that start an episode in it (a task may add to it)"""

    def _after_device_step(self, resetting):
        """host-side task state taken from the record of the device step just taken"""

    def step_device(self, action):
        """Device-resident control step for a policy that lives on the GPU: `action` is a CUDA tensor / array exposing
        `__cuda_array_interface__` (fp32, [n_envs, n_action], on this env's device); returns zero-copy torch views
        (observation rows [n_envs, obs_dim], out [n_envs, 4] = reward, discount, step_type, 0) of the library's buffers, valid
        until the next step.  Nothing is copied to the host and the call does not synchronise: work is ordered on
        `env.physics.stepper.stream` (wrap it in `torch.cuda.ExternalStream` to order a policy after it).  Requires
        `device_task=True`; `observation_layout()` names the columns.  With a dataset the envs that reset draw their trajectory (and,
        flight, start step) on the device (counter hash of seed, env, episode), so no trajectory index may be pending."""
        if not self._device_task:
            raise RuntimeError('step_device needs device_task=True (task hooks on the device)')
        self._launch_step_device(action)
        return self._device_views()

    def _launch_step_device(self, action):
        """the work of step_device up to its result views: the control step on the device, for actions already there (nothing read back)"""
        self._ensure_programs()
        cai = action.__cuda_array_interface__
        assert tuple(cai['shape']) == (self.n_envs, self._action_spec.shape[0]) and cai['typestr'] == '<f4', cai
        self._sim.task_step(cai['data'][0], self._n_sub, is_device=True)
        self._needs_reset[:] = False            # (host mirror of the device's reset flags: not read back on this path)

    def _device_views(self):
        """zero-copy torch views (observation rows [n_envs, obs_dim], out [n_envs, 4]) of the library's task buffers"""
        if self._dev_views is None:
            obs_ptr, dim, out_ptr = self._sim.task_ptrs()
            self._dev_views = (_device_tensor(obs_ptr, (self.n_envs, dim), '<f4', self._sim.device),
                               _device_tensor(out_ptr, (self.n_envs, 4), '<f4', self._sim.device))
        return self._dev_views

    def _unbatch(self, ts, first=False):
        if self._batched:
            return ts
        obs = collections.OrderedDict((k, v[0]) for k, v in ts.observation.items())
        if first or ts.step_type[0] == StepType.FIRST:
            return TimeStep(StepType.FIRST, None, None, obs)
        return TimeStep(StepType(int(ts.step_type[0])), float(ts.reward[0]), float(ts.discount[0]), obs)

    # ----------------------------------------------------------------------------- state rows
    # physics.get_state() / set_state() for the envs of the batch, with everything the task carries per env (fb_state_* in the header).
    # The device keeps a bank of rows; the env object's own per-env arrays that shape the coming outputs (`_state_refs`) are kept per
    # bank slot in a host-side mirror.  Not covered, NotImplementedError: the host-side task code with a trajectory dataset (per-env
    # snippets and their feature bank live in Python objects) and the host-side vision task (per-env terrains).  One limit: with the
    # task on the device the draws of a reset are a counter hash of (seed, env, episode), so a row loaded into another env id
    # continues bit for bit until that env's next reset, whose draws follow the new id.
    def _state_refs(self):
        """(owner, attribute) of the per-env host arrays a state row goes with"""
        return [(self, '_time'), (self, '_needs_reset')]

    def _state_prepare(self):
        """the programs that shape the row are on the device (a fresh env uploads them at its first reset)"""
        self._ensure_programs()

    def state_bank(self, n_slots):
        """(re)allocate the bank of `n_slots` state rows on the device and its host-side mirror (0 frees them).  Replacing the env's
        programs (a new shared reference trajectory, `enable_eyes` does not) drops the bank: allocate it again afterwards."""
        self._state_prepare()
        self._sim.state_bank(n_slots)
        self._state_mirror = [np.zeros((int(n_slots),) + getattr(o, a).shape[1:], getattr(o, a).dtype) for o, a in self._state_refs()]

    def _state_ids(self, slots, env_ids):
        if slots is None and env_ids is None:
            env_ids = np.arange(self.n_envs)
        e = np.arange(len(np.atleast_1d(slots))) if env_ids is None else np.asarray(env_ids, np.int64).reshape(-1)
        s = np.arange(len(e)) if slots is None else np.asarray(slots, np.int64).reshape(-1)
        if getattr(self, '_state_mirror', None) is None:
            raise RuntimeError('no state bank: call state_bank(n_slots) first')
        return s, e

    def save_state(self, slots=None, env_ids=None):
        """env `env_ids[k]` -> bank slot `slots[k]` (None: 0 .. n - 1; both None: every env k -> slot k).  Nothing leaves the device
        and the call does not synchronise."""
        s, e = self._state_ids(slots, env_ids)
        self._sim.save_state(s, e)
        for buf, (o, a) in zip(self._state_mirror, self._state_refs()):
            buf[s] = getattr(o, a)[e]

    def load_state(self, slots=None, env_ids=None):
        """bank slot `slots[k]` -> env `env_ids[k]` (None: 0 .. n - 1); one slot may feed many envs, an env may appear once, the other
        envs are untouched.  The views `step_device` returned and the next `step()` see the saved rows.  The env's RandomStates (the host
        draws of later resets) are not part of a slot: `state_dict()` carries them."""
        s, e = self._state_ids(slots, env_ids)
        self._sim.load_state(s, e)
        for buf, (o, a) in zip(self._state_mirror, self._state_refs()):
            arr = np.array(getattr(o, a))
            arr[e] = buf[s]
            setattr(o, a, arr)

    def _state_rngs(self):
        """the RandomStates a continuation draws from, by name"""
        return {'env': self._rs}

    def state_dict(self):
        """Every env's state as plain numpy arrays and ints (np.savez and pickle work): the rows of all envs, the layout signature, the
        host-side mirror, the counters and the RandomStates.  Uses slots 0 .. n_envs - 1 of the bank (allocated if there is none)."""
        self._state_prepare()
        if getattr(self, '_state_mirror', None) is None or len(self._state_mirror[0]) < self.n_envs:
            self.state_bank(self.n_envs)
        self.save_state()
        d = {'signature': np.uint64(self._sim.state_signature()), 'rows': self._sim.read_states(np.arange(self.n_envs)),
             'nsub_done': self._sim.state_substeps(), 'n_resets': int(self.n_resets), 'n_capacity_overflows': int(self.n_capacity_overflows)}
        for k, (o, a) in enumerate(self._state_refs()):
            d[f'host_{k}{a}'] = np.array(getattr(o, a))
        for name, rs in self._state_rngs().items():
            _, keys, pos, has_gauss, cached = rs.get_state()
            d[f'rng_{name}_keys'], d[f'rng_{name}_pos'] = np.array(keys), int(pos)
            d[f'rng_{name}_has_gauss'], d[f'rng_{name}_cached'] = int(has_gauss), float(cached)
        return d

    def load_state_dict(self, d):
        """continue from a `state_dict()` of an env built the same way (same factory arguments: the layout signature must match)"""
        self._state_prepare()
        if int(d['signature']) != self._sim.state_signature():
            raise ValueError(f"state_dict signature {int(d['signature']):#x} does not match this env's state layout "
                             f'{self._sim.state_signature():#x}: the model, the programs or the reference slot length differ')
        rows = np.asarray(d['rows'])
        if rows.shape[0] != self.n_envs:
            raise ValueError(f'state_dict holds {rows.shape[0]} envs, this env has {self.n_envs}')
        if getattr(self, '_state_mirror', None) is None or len(self._state_mirror[0]) < self.n_envs:
            self.state_bank(self.n_envs)
        ids = np.arange(self.n_envs)
        self._sim.write_states(ids, rows)
        for k, (buf, (o, a)) in enumerate(zip(self._state_mirror, self._state_refs())):
            buf[ids] = np.asarray(d[f'host_{k}{a}'])
        self.load_state(ids, ids)
        self._sim.state_substeps(int(d['nsub_done']))
        self.n_resets, self.n_capacity_overflows = int(d['n_resets']), int(d['n_capacity_overflows'])
        for name, rs in self._state_rngs().items():
            rs.set_state(('MT19937', np.asarray(d[f'rng_{name}_keys'], np.uint32), int(d[f'rng_{name}_pos']),
                          int(d[f'rng_{name}_has_gauss']), float(d[f'rng_{name}_cached'])))

    def close(self):
        self._sim.close()


class BatchedFlyEnv(_TaskEnv):
    """dm_env-shaped environment over N lock-stepped FruitFly walkers (composer.Environment stand-in): the walker's observables, its eye
    cameras, applied forces and reset noise.  The tasks are `TemplateTaskEnv`, `WalkOnBallEnv`, `WalkImitationEnv` and
    `FlightImitationEnv`; each names its model (`flymodel.load_model`) in `_MODEL`."""
    _MODEL = None

    def __init__(self, n_envs, time_limit, device=0, lib_path=None, reset_noise=0.0, seed=0, device_task=False, model=None):
        # `model`: a variant from flymodel.model_for
        super().__init__(model if model is not None else load_model(self._MODEL), n_envs, device, lib_path, time_limit, seed, device_task)
        m = self.model
        self._device = int(device)
        self.physics = _PhysicsFacade(self)
        self._reset_noise = reset_noise
        sn, sens = m.meta['site_names'], m.meta['sensor_names']

        def sd(names_):
            out = []
            for n_ in names_:
                i = sens.index('walker/' + n_)
                out.extend(range(m.sensor_adr[i], m.sensor_adr[i] + m.sensor_dim[i]))
            return np.array(out)
        self._sd = dict(accelerometer=sd(['accelerometer']), gyro=sd(['gyro']), velocimeter=sd(['velocimeter']))
        self._has_legs = 'walker/force_tarsus_T1_left' in sens      # Walking always; Flying with disable_legs=False (base.py:360-364)
        if self._has_legs:
            legs = [f'T{k}_{s}' for k in (1, 2, 3) for s in ('left', 'right')]
            self._sd.update(force=sd([f'force_tarsus_{l}' for l in legs]), touch=sd([f'touch_claw_{l}' for l in legs]))
            app = [f'walker/claw_T{k}_{s}' for k in (1, 2, 3) for s in ('left', 'right')] + ['walker/head']
            self._app_sites = np.array([sn.index(n) for n in app])
        else:
            self._app_sites = np.zeros(0, np.int64)
        self._leg_act_qadr = np.array([m.jnt_qposadr[m.actuator_trnid[i]] for i in range(m.nu)
                                       if m.actuator_trntype[i] == 0 and any(t in m.meta['actuator_names'][i] for t in ('T1', 'T2', 'T3'))],
                                      np.int64)

    # ---------------------------------------------------------------------------------- specs
    def _obs_table(self):
        """(name, width, shape, program item) per observable in spec order, hidden entries last, and the index lists the items read: the
        walker's appendage sites, observable joints' qpos and qvel addresses, then the task's (`_task_obs`)."""
        m, sd = self.model, self._sd
        nq, napp = len(self._obs_qadr), len(self._app_sites)
        o_app, o_q, o_v = 0, napp, napp + nq
        items, hidden, lists = self._task_obs(napp + 2 * nq)
        items |= {
            'accelerometer': (3, (3,), (st.OBS_SENSOR_MEAN, sd['accelerometer'][0], 3)),
            'actuator_activation': (m.na, (m.na,), (st.OBS_ACT, 0, m.na)),
            'appendages_pos': (3 * napp, (3 * napp,), (st.OBS_SITES_EGO, o_app, napp)),
            'gyro': (3, (3,), (st.OBS_SENSOR_MEAN, sd['gyro'][0], 3)),
            'joints_pos': (nq, (nq,), (st.OBS_QPOS, o_q, nq)),
            'joints_vel': (nq, (nq,), (st.OBS_QVEL, o_v, nq)),
            'velocimeter': (3, (3,), (st.OBS_SENSOR_MEAN, sd['velocimeter'][0], 3)),
            'world_zaxis': (3, (3,), (st.OBS_ROOT_ZAXIS, 0, 3)),
        }
        if 'force' in sd:
            items['force'] = (len(sd['force']), (len(sd['force']),), (st.OBS_SENSOR_MEAN, sd['force'][0], len(sd['force'])))
            items['touch'] = (len(sd['touch']), (len(sd['touch']),), (st.OBS_SENSOR_MEAN, sd['touch'][0], len(sd['touch'])))
        names = list(self._OBS)
        if self._has_legs and 'force' not in names:      # Flying with legs: appendages_pos, force, touch join the walker's observables,
            walker = sorted(names[:-2] + ['appendages_pos', 'force', 'touch'])      # which dm_control lists alphabetically, task ones last
            names = walker + names[-2:]
        rows = [('walker/' + k,) + items[k] for k in names]
        rows += [('_velocimeter_now', 3, (3,), (st.OBS_SENSOR_NOW, sd['velocimeter'][0], 3)),
                 ('_gyro_now', 3, (3,), (st.OBS_SENSOR_NOW, sd['gyro'][0], 3)),
                 ('_scalars', 3, (3,), (st.OBS_SCALARS, 0, 3))]
        return rows + hidden, list(self._app_sites) + list(self._obs_qadr) + list(self._obs_vadr) + lists

    def _task_obs(self, o):
        """the task's observables {name: (width, shape, program item)}, its hidden rows and the index lists they read, which start at `o`"""
        return {}, [], []

    def observation_spec(self):
        lead = (self.n_envs,) if self._batched else ()
        return collections.OrderedDict((n, Array(lead + shp, np.float32, name=n)) for n, _, shp, _ in self._obs_table()[0]
                                       if not n.startswith('_'))

    def observation_layout(self):
        """{observable name: (column slice, shape)} of the observation rows `step_device` returns."""
        return {k: (sl, self._obs_shapes[k]) for k, sl in self._obs_slices.items() if not k.startswith('_')}

    # -------------------------------------------------------------------------------- episode
    def _upload_program(self):
        """Observation program = the task's observables in spec order, evaluated on the device (fb_obs_program); with the task hooks on
        the device also the task program."""
        self._upload_obs_program(*self._obs_table())
        if self._device_task:
            self._upload_task_program()
            self._dev_views = None

    def _upload_task_program(self):
        """fb_task_program: the task hooks of this env as a device-side program (same constants as the host path)."""
        self._sim.task_program(**self._task_program())

    def _ensure_programs(self):
        if self._rec is None:
            self._upload_program()

    def _before_step(self, action, resetting):
        """the host's before_step -> (the rows set_control takes, their host -> device bytes).  Here the actions as they are: the device
        action map permutes them into ctrl and zeroes NaN."""
        return action, action.nbytes

    def _state_refs(self):
        return super()._state_refs() + [(self, '_step_counter')]

    def set_applied_forces(self, qfrc=None, xfrc=None, env_ids=None):
        """MuJoCo's `physics.data.qfrc_applied` ([nv] per env) and `xfrc_applied` ([nbody, 6] per env: world-frame force, then torque,
        at each body's CoM) for every env (`env_ids` None; a single row broadcasts) or the listed envs.  They act in every physics
        substep until overwritten or cleared, and a reset of an env zeroes its own (mj_resetData).  None leaves a field as it is.
        The batched counterpart of writing them from a per-substep `mjcb_control` callback."""
        self._sim.set_applied(qfrc, xfrc, env_ids)

    def clear_applied_forces(self):
        """zero every env's applied forces (the step goes back to the path without the applied-force term)"""
        self._sim.clear_applied()

    def set_model_params(self, env_ids=None, **fields):
        """`physics.model` writes without mj_setConst, per env: fields named as mjModel's (`stepper.PARAMS`: body_mass [nbody],
        body_inertia [nbody, 3], dof_armature, dof_damping [nv], jnt_stiffness [njnt], geom_friction [ngeom, 3], actuator_gainprm,
        actuator_biasprm [nu, 3] (MuJoCo's first three entries), gravity, wind [3], density, viscosity [1]) for every env (`env_ids`
        None; a single row broadcasts) or the listed envs.  They persist across steps and resets until overwritten or cleared."""
        for name, v in fields.items():
            self._sim.param_set(name, v, env_ids)

    def model_params(self):
        """-> {field: [n_envs, ...] float32} of every per-env model parameter (the compiled values where none was set)"""
        m = self.model
        shapes = {'body_inertia': (m.nbody, 3), 'geom_friction': (m.ngeom, 3), 'actuator_gainprm': (m.nu, 3), 'actuator_biasprm': (m.nu, 3)}
        return {name: self._sim.param_get(name).reshape((self.n_envs,) + shapes.get(name, (-1,))) for name in st.PARAMS}

    def randomize_model_params(self, seed=0, shared=(), **ranges):
        """domain randomisation: at every reset of an env from now on, each named field is drawn from U(lo, hi) per element (`name=(lo,
        hi)`, each broadcast to the field's shape), or with one draw for all its elements for the names in `shared` (lo = 0.8 m,
        hi = 1.2 m scales every element by one factor).  Draws are a counter hash of (seed, env, the env's reset count, field, element):
        the same on the host-side and the device-side task code.  Fields not named keep their values."""
        for name in shared:
            if name not in ranges:
                raise ValueError(f'shared names {name!r}, which has no range')
        for name, (lo, hi) in ranges.items():
            self._sim.param_draws(name, lo, hi, shared=name in shared, seed=seed)

    def clear_model_params(self):
        """every env back to the compiled model's parameters, and no draws (the step goes back to the model's tables)"""
        self._sim.param_clear()

    def set_reset_noise(self, amp):
        """U(-amp, amp) rad added to the actuated leg joints of the start pose at the resets from now on (0: the reference's exact
        start pose).  `reset_noise=` of the factory sets the initial value; a batch is typically started with noise once, so that the
        envs decorrelate, and reset exactly afterwards."""
        if self._device_task and amp > 0 and not self._reset_noise > 0:
            raise ValueError('the device task program was uploaded without a noise joint list: create the env with reset_noise > 0')
        if self._device_task:
            self._sim.task_set_reset_noise(amp)
        else:
            self._reset_noise = float(amp)

    def device_reset_count(self):
        """episodes started so far, summed over the envs (device-side task logic: read from the device's episode counters)"""
        return int(self._sim.task_episodes().sum()) if self._device_task else int(self.n_resets)

    # ---------------------------------------------------------------------------------- eyes
    def enable_eyes(self, size=32, fovy=150.0, terrain_shape=None, half_size=20.0, z_offset=0.0):
        """Turn on the eye-camera observables `walker/right_eye`, `walker/left_eye` (reference `fruitfly.py:729-745`; 32 x 32,
        fovy 150 in `tasks/vision_flight.py:23-24`), rendered on the device by a ray caster over an optional per-env
        heightfield `terrain_shape = (nrow, ncol)` spanning [-half_size, half_size]^2 (`flybody_b200.arenas`), the ground plane
        and a sky.  `render_eyes()` returns them for the current state; they are not part of `step()`'s observation dict."""
        nrow, ncol = terrain_shape if terrain_shape is not None else (0, 0)
        self._eye_program(size, fovy, nrow, ncol, half_size, z_offset)
        self._eyes_on = True

    def set_terrain(self, env_ids, heights):
        """heights [n, nrow, ncol] (world units; row = y, col = x) of the listed envs' terrains, as seen by the eyes."""
        self._sim.hfield_write(env_ids, heights)

    def render_eyes(self):
        """OrderedDict {'walker/right_eye', 'walker/left_eye'}: uint8 [n_envs, size, size, 3] from the current poses."""
        if not getattr(self, '_eyes_on', False):
            raise RuntimeError('call enable_eyes() first')
        img = self._sim.render_eyes()
        return collections.OrderedDict((name, img[:, k]) for k, (name, _, _) in enumerate(_EYE_CAMERAS))

    # ---------------------------------------------------------------------------- observations
    def _observation(self, rec):
        """Views into the device-evaluated observation rows (fp32; the reference returns float64 copies)."""
        N = self.n_envs
        obs = collections.OrderedDict()
        for k, sl in self._obs_slices.items():
            if not k.startswith('_'):
                obs[k] = rec[:, sl].reshape((N,) + self._obs_shapes[k])
        return obs


class TemplateTaskEnv(BatchedFlyEnv):
    """Batched `TemplateTask` (reference `tasks/template_task.py`): the walker on the flat Walking floor without a ghost or a
    reference.  Every episode starts from the template pose at rest (`qpos0`, the upright spawn); the reward is 1; an episode ends
    early only on a bad state (non-finite, or |qacc| > _TERMINAL_QACC: base.py:222-225, discount 0), else at the time limit (discount 1).
    An optional `action_corruptor(action, random_state)` rewrites the actions on the host before they are applied; `prev_action`
    returns what was applied (the reference walker's `prev_action`)."""
    _MODEL, _CONTROL_TIMESTEP, _KIND, _OBS, _TASK = 'template', _WALK_CONTROL_TIMESTEP, st.TASK_TEMPLATE, _WALKER_OBS, TemplateTask

    def __init__(self, n_envs, time_limit=1.0, action_corruptor=None, random_state=None, **kw):
        super().__init__(n_envs, time_limit, **kw)
        self.task = self._TASK(self, time_limit, self._control_timestep)
        self._corruptor = action_corruptor
        if random_state is not None:
            self._rs = random_state if isinstance(random_state, np.random.RandomState) else np.random.RandomState(random_state)
        self._prev_action = np.zeros((self.n_envs, self._action_spec.shape[0]))

    def _state_refs(self):
        return super()._state_refs() + [(self, '_prev_action')]

    @property
    def prev_action(self):
        """the actions applied by the last step (after the corruptor; zero for an env that started an episode in it)"""
        return self._prev_action.copy() if self._batched else self._prev_action[0].copy()

    def _action(self, action):
        action = super()._action(action, host=True)
        if self._corruptor is not None:                 # before_step (template_task.py): on the host, before the action map
            action = np.array(self._corruptor(action, self._rs), np.float64).reshape(self.n_envs, -1)
        self._prev_action = np.where(self._needs_reset[:, None], 0.0, action)      # a resetting env drops its action (composer auto-reset)
        return action.astype(np.float32)

    def _reset_envs(self, ids, hold=False):
        """physics.reset() (mj_resetData: qpos0 at rest, controls and applied forces zeroed) + initialize_episode"""
        ids = np.asarray(ids)
        self._ensure_programs()
        self._start_episodes(ids, np.tile(self.model.qpos0, (len(ids), 1)), None, hold)
        self._prev_action[ids] = 0.0

    def _before_device_step(self, resetting):
        self._prev_action[resetting] = 0.0

    def _task_after(self, rec, obs, resetting, time, ghost):
        """get_reward (factors (1,)), check_termination (base.py:222-225), get_discount; the device task FB_TASK_TEMPLATE is the same
        logic"""
        return self._end_step(resetting, self._bad_state(rec), 1.0, time)

    def step_device(self, action):
        if self._corruptor is not None:
            raise RuntimeError('step_device does not run an action_corruptor (a host callable): corrupt the actions on the device, '
                               'or use step()')
        return super().step_device(action)


_BALL_TARGET_QVEL = (0.0, -5.0, 0.0)            # target ball angular velocity of walk_on_ball (tasks/walk_on_ball.py:67)
_BALL_MARGIN = 6.0                              # ... and the margin of its linear tolerance


class WalkOnBallEnv(TemplateTaskEnv):
    """Batched `WalkOnBall` (reference `tasks/walk_on_ball.py`, `tasks/arenas/ball.py`): the fly tethered at its spawn pose (thorax
    welded to the world) walks on a floating ball.  Every episode starts from `qpos0` at rest (mj_resetData: the ball's quaternion is
    the identity).  The reward is the product over the ball's three angular velocities of max(0, 1 - |ball_qvel - (0, -5, 0)| / 6);
    an episode ends with discount 0 when |velocimeter| > 50, |gyro| > 200 or the state is bad (non-finite, |qacc| > 1e14), and with
    discount 1 at the 2 s time limit.  `before_step` applies the action only."""
    # the walker's observables, then the task's ball_qvel (reference tasks/walk_on_ball.py:46)
    _MODEL, _KIND, _OBS, _TASK = 'ball', st.TASK_BALL, _WALKER_OBS + ('ball_qvel',), WalkOnBallTask

    def __init__(self, n_envs, time_limit=2.0, **kw):
        super().__init__(n_envs, time_limit=time_limit, **kw)
        self._ball_v = self.model.jnt_dofadr_of('ball')

    def _task_obs(self, o):
        # qvel of the ball joint after the last substep
        return {'ball_qvel': (3, (3,), (st.OBS_QVEL, o, 3))}, [], list(range(self._ball_v, self._ball_v + 3))

    def _task_program(self):
        return super()._task_program() | dict(terminal_linvel=_TERMINAL_LINVEL, terminal_angvel=_TERMINAL_ANGVEL, ball_vadr=self._ball_v,
                                              ball_target=_BALL_TARGET_QVEL, ball_margin=_BALL_MARGIN)

    def _task_after(self, rec, obs, resetting, time, ghost):
        """get_reward_factors, check_termination (walk_on_ball.py:55-81, base.py:222-225), get_discount; the device task FB_TASK_BALL is
        the same logic"""
        sl = self._obs_slices
        linvel = np.linalg.norm(rec[:, sl['_velocimeter_now']], axis=1)
        angvel = np.linalg.norm(rec[:, sl['_gyro_now']], axis=1)
        terminate = (linvel > _TERMINAL_LINVEL) | (angvel > _TERMINAL_ANGVEL) | self._bad_state(rec)
        ball_qvel = obs['walker/ball_qvel'].astype(np.float64)
        reward = np.prod(linear_tolerance(ball_qvel - np.asarray(_BALL_TARGET_QVEL), _BALL_MARGIN), axis=1)
        return self._end_step(resetting, terminate, reward, time)


class _ImitationEnv(BatchedFlyEnv):
    """The walker tracking a reference trajectory with a ghost (walk_imitation, flight_imitation): one reference shared by all envs (the
    Inference* loaders hold a single trajectory) or one per env (dataset loaders hand out a different snippet per episode), on the host or,
    for a dataset with the task on the device, cut from a device bank of the whole dataset."""

    def __init__(self, n_envs, terminal_com_dist, time_limit, future_steps, traj_generator=None, inference_mode=True,
                 max_reference_steps=None, **kw):
        super().__init__(n_envs, time_limit, **kw)
        m, N = self.model, self.n_envs
        self.task = self._TASK(self, traj_generator or self._LOADER(), terminal_com_dist, future_steps, time_limit, self._control_timestep)
        self._ghost_q, self._ghost_v = m.jnt_qposadr_of('ghost/'), m.jnt_dofadr_of('ghost/')
        self._future = future_steps + 1
        self._program_ref_id = None
        self._program_switched = False
        # the shared case keeps one device table, the per-env case one slot per env
        tg = self.task._traj_generator
        self._per_env_ref = not isinstance(tg, (InferenceWalkingTrajectoryLoader, InferenceFlightTrajectoryLoader))
        self._max_reference_steps = max_reference_steps
        self._ref_rows = None                       # per-env mode: [N, slot_len, 13] fp32 (root qpos 7, root qvel 6), padded with the last row
        self._ref_len = np.zeros(N, np.int64)
        self._episode_steps = np.zeros(N, np.int64)
        self._ref_pick = np.zeros((N, 2), np.int64)      # dataset on the device: (trajectory, start step) the host pinned last
        self._bank_rows = None                           # ... and the dataset as uploaded by fb_ref_bank (_bank_tables)
        self._ref_qpos = None
        # full-body imitation reward (reference walk_imitation.py:152-177): mocap joints / sites named by the dataset
        self._inference_mode = bool(inference_mode)
        # a trajectory dataset on the device: the whole dataset in a device bank, every reset cuts its own reference from it
        self._device_bank = self._device_task and self._per_env_ref and isinstance(tg, (HDF5FlightTrajectoryLoader, HDF5WalkingTrajectoryLoader))
        if self._device_task and not self._device_bank and (self._per_env_ref or not self._inference_mode):
            raise NotImplementedError('device_task covers the shared-reference (inference-mode) tasks and the HDF5 trajectory datasets of '
                                      'walk_imitation / flight_imitation')

    def _task_obs(self, o):
        f = self._future
        return {'ref_displacement': (3 * f, (f, 3), (st.OBS_REF_DISP, 0, f)), 'ref_root_quat': (4 * f, (f, 4), (st.OBS_REF_QUAT, 0, f))}, [], []

    def _upload_obs_program(self, rows, lists):
        """... with the reference the ref_* observables read: the shared trajectory, or one slot per env (`ref_slot_write`)"""
        super()._upload_obs_program(rows, lists, np.zeros((self._future, 7)) if self._per_env_ref else self._ref_qpos[:, :7])
        if self._per_env_ref:
            self._sim.ref_slots(self._slot_len)

    def _task_program(self):
        t, sl = self.task, self._obs_slices
        kw = super()._task_program() | dict(
            ghost_qadr=self._ghost_q, ghost_vadr=self._ghost_v, ghost_offset=t._ghost_offset, terminal_com_dist=min(t._terminal_com_dist, 3e38),
            terminal_linvel=_TERMINAL_LINVEL, terminal_angvel=_TERMINAL_ANGVEL, terminal_height=_TERMINAL_HEIGHT,
            obs_refdisp_off=sl['walker/ref_displacement'].start, obs_refquat_off=sl['walker/ref_root_quat'].start, com_offset=_COM_OFFSET)
        if self._device_bank:                   # the draws of _load_snippet, then the task's own use of the bank (_bank_program)
            tg = t._traj_generator
            kw.update(ref_bank=1, n_pick=len(tg.traj_indices), pick_traj=np.asarray(tg.traj_indices, np.int64), future_steps=t._future_steps,
                      **self._bank_program())
        else:
            kw.update(episode_steps=int(self._steps_of(self._ref_qpos.shape[0])), ref_len=self._ref_qpos.shape[0], ref_qpos=self._ref_qpos[:, :7],
                      ref_qvel=self._ref_qvel[:, :6])
        return kw

    def _ensure_programs(self):
        if self._rec is None:
            if self._device_bank:               # (the references are drawn by the resets)
                self._ensure_slots()
            else:
                self._load_snippet(np.arange(self.n_envs))

    def _load_snippet(self, ids):
        """initialize_episode_mjcf: pick the reference of the episode that starts now (walk_imitation.py:93-110,
        flight_imitation.py:88-111).  Shared mode: ONE trajectory for every env, re-uploaded when the loader returns different
        values (content digest, so in-place edits count).  The switch is global: envs in mid-episode follow the new trajectory from
        their current step on, and with the task hooks on the device the re-upload restarts every env (`_program_switched`) -- a
        batch whose envs need independent references uses the per-env mode (`ref_path=` datasets), where each env of `ids` draws
        its own snippet and only its device slot is rewritten (with the task on the device: the device cuts the snippet from
        its trajectory bank, `_pick_references`)."""
        t = self.task
        tg = t._traj_generator
        if not self._per_env_ref:
            snip = tg.get_trajectory(traj_idx=t._next_traj_idx)
            t._next_traj_idx = None
            qpos, qvel = self._snippet_root(snip)
            qpos, qvel = np.asarray(qpos, np.float64), np.asarray(qvel, np.float64)
            key = (qpos.shape, hashlib.blake2b(qpos.tobytes() + qvel.tobytes(), digest_size=16).digest())
            if self._program_ref_id != key:
                self._program_switched = self._program_ref_id is not None
                self._program_ref_id = key
                self._ref_qpos, self._ref_qvel = qpos, qvel
                self._upload_program()
            self._ref_len[:] = self._ref_qpos.shape[0]
            self._episode_steps[:] = self._steps_of(self._ref_qpos.shape[0])
            return
        self._ensure_slots()
        if self._device_bank:
            self._pick_references(ids)
            return
        L = self._slot_len
        for e in ids:
            idx = t._next_traj_idx
            if idx is None and hasattr(tg, 'traj_indices') and hasattr(tg, '_random_state'):
                idx = tg._random_state.choice(tg.traj_indices)             # the draw the loader itself would make
            snip = tg.get_trajectory(traj_idx=idx)
            qpos, qvel = self._snippet_root(snip)
            n = min(qpos.shape[0], L)
            self._ref_rows[e, :n, :7], self._ref_rows[e, :n, 7:] = qpos[:n], qvel[:n]
            self._ref_rows[e, n:] = self._ref_rows[e, n - 1]
            self._ref_len[e] = n
            self._episode_steps[e] = self._steps_of(n)
            if not self._inference_mode:
                self._env_bank_off[e] = self._bank.offset_of(idx, snip)
        t._next_traj_idx = None
        self._sim.ref_slot_write(ids, self._ref_rows[ids, :, :7])

    def _ensure_slots(self):
        """per-env mode: the slot length (the longest reference an episode can consume), the host mirror and the programs, once"""
        if self._ref_rows is not None:
            return
        t, tg = self.task, self.task._traj_generator
        cap = self._max_reference_steps or (t._max_episode_steps + t._future_steps + 1)
        if hasattr(tg, 'trajectory_len') and hasattr(tg, 'num_trajectories'):
            cap = min(cap, max(int(tg.trajectory_len(i)) for i in range(tg.num_trajectories)))
        self._slot_len = int(cap)
        self._ref_rows = np.zeros((self.n_envs, self._slot_len, 13), np.float32)
        self._upload_program()

    def _bank_tables(self):
        """(rows per trajectory, rows [sum][w]) of every trajectory of the dataset for the device bank (`_bank_rows_of`) -- all of them,
        because set_next_trajectory_index may name any.  Kept as the host mirror's source."""
        if self._bank_rows is None:
            tg = self.task._traj_generator
            rows = [self._bank_rows_of(j) for j in range(tg.num_trajectories)]
            self._bank_len = np.asarray([r.shape[0] for r in rows], np.int64)
            self._bank_off = np.concatenate([[0], np.cumsum(self._bank_len)[:-1]]).astype(np.int64)
            self._bank_rows = np.concatenate(rows, 0).astype(np.float32)
        return self._bank_len, self._bank_rows

    def _pick_references(self, ids):
        """dataset with the task on the device: the draws the host-side code makes at these resets (ascending env id; from the
        loader's RandomState `choice`, then, flight, `randint`; a pending set_next_trajectory_index goes to every env of `ids` and is
        then cleared), pinned for the device's reset (fb_task_ref_pick).  The host mirror (_ref_rows, _ref_len, _episode_steps;
        walking: _env_bank_off into the feature mirror) is cut from the bank as ktask_reset_ref cuts it: fp32 rows start .. start + n,
        root x, y relative to the x, y in columns 13, 14 of row `start` (flight: the CoM's, walking: the root's), padded with the last row."""
        t, tg = self.task, self.task._traj_generator
        ids = np.sort(np.asarray(ids, np.int64))
        traj, start = np.zeros(len(ids), np.int64), np.zeros(len(ids), np.int64)
        random_start = getattr(tg, 'randomize_start_step', False)      # walking snippets always start at row 0
        for k in range(len(ids)):
            idx = t._next_traj_idx
            if idx is None:
                idx = tg._random_state.choice(tg.traj_indices)
            traj[k] = idx
            start[k] = tg._random_state.randint(tg.trajectory_len(idx) - tg.START_MARGIN) if random_start else 0
        t._next_traj_idx = None
        self._sim.task_ref_pick(ids, traj, start)
        self._ref_pick[ids, 0], self._ref_pick[ids, 1] = traj, start
        for e, j, s0 in zip(ids, traj, start):
            rows = self._bank_rows[self._bank_off[j] + s0:self._bank_off[j] + self._bank_len[j]]
            n = min(rows.shape[0], self._slot_len)
            r = rows[:n, :13].copy()
            r[:, :2] -= rows[0, 13:15]
            self._ref_rows[e, :n], self._ref_rows[e, n:] = r, r[n - 1]
            self._ref_len[e] = n
            self._episode_steps[e] = self._steps_of(n)
        if not self._inference_mode:
            self._env_bank_off[ids] = self._bank_off[traj]

    def reference_picks(self):
        """(trajectory index, start step) of the reference every env tracks in its running episode, int32 [n_envs] each, read from
        the device (walk_imitation / flight_imitation with a dataset and device_task=True; walking starts at 0) -- e.g. to log which
        trajectory each env follows."""
        if not self._device_bank:
            raise RuntimeError('reference_picks needs walk_imitation / flight_imitation(ref_path=..., device_task=True)')
        if self._rec is None:
            raise RuntimeError('no episode has started yet: call reset() or step_device() first')
        traj, start = self._sim.task_ref_state()
        return (traj, start) if self._batched else (int(traj[0]), int(start[0]))

    def _ref_at(self, step, ids=None):
        """[n, 13] root reference (qpos 7, qvel 6) of the listed envs at their own steps."""
        if not self._per_env_ref:
            return np.concatenate([self._ref_qpos[step, :7], self._ref_qvel[step, :6]], 1)
        ids = np.arange(self.n_envs) if ids is None else ids
        return self._ref_rows[ids, step].astype(np.float64)

    def _reset_envs(self, ids, hold=False):
        """initialize_episode: the root on the reference's first row and the ghost placed on it, then the task's start pose (`_start_pose`)"""
        m = self.model
        ids = np.asarray(ids)
        self._load_snippet(ids)
        n = len(ids)
        qpos = np.tile(m.qpos0, (n, 1))
        ref0 = self._ref_at(np.zeros(n, np.int64), ids)
        qpos[:, self._root_q:self._root_q + 7] = ref0[:, :7]
        qpos[:, self._ghost_q:self._ghost_q + 7] = ref0[:, :7] + np.concatenate([self.task._ghost_offset, np.zeros(4)])
        self._start_episodes(ids, qpos, self._start_pose(ids, qpos, ref0), hold)

    def _before_step(self, action, resetting):
        # before_step (walk_imitation.py:138-150, flight_imitation.py:146-168, base.py:197-201): the ghost on the reference row of the step
        step = np.round(self._time / self._control_timestep).astype(np.int64)
        step = np.minimum(step, self._ref_len - 1)
        step = np.where(resetting, 0, step)
        ghost = self._ref_at(step)
        ghost[:, :3] += self.task._ghost_offset
        ghost = ghost.astype(np.float32)
        ghost[resetting, 7:] = 0.0
        self._sim.write_state(st.QPOS, np.arange(self._ghost_q, self._ghost_q + 7), ghost[:, :7])
        self._sim.write_state(st.QVEL, np.arange(self._ghost_v, self._ghost_v + 6), ghost[:, 7:])
        ctrl, nbytes = super()._before_step(action, resetting)
        return ctrl, nbytes + ghost.nbytes

    def _before_device_step(self, resetting):
        if resetting.any():
            self._load_snippet(np.nonzero(resetting)[0])            # a trajectory set since the last reset re-uploads the programs
            if self._program_switched:                              # ... which restarts every env on the device (fb_task_reset_all)
                resetting[:] = True
                self._program_switched = False

    def _state_refs(self):
        return super()._state_refs() + [(self, '_ref_len'), (self, '_episode_steps'), (self, '_ref_pick')]

    def _state_prepare(self):
        if self._per_env_ref and not self._device_bank:
            raise NotImplementedError('state rows do not cover the host-side task code with a trajectory dataset (per-env snippets are '
                                      'Python objects): use device_task=True')
        super()._state_prepare()

    def _state_rngs(self):
        rngs = super()._state_rngs()
        tg = self.task._traj_generator
        if isinstance(getattr(tg, '_random_state', None), np.random.RandomState):
            rngs['loader'] = tg._random_state
        return rngs

    def _launch_step_device(self, action):
        if self._device_bank and self.task._next_traj_idx is not None:
            raise RuntimeError('set_next_trajectory_index is pending: which envs reset next is only known on the device, so apply it '
                               'with step() (every env resetting in that step gets the index)')
        super()._launch_step_device(action)


class WalkImitationEnv(_ImitationEnv):
    """Batched `WalkImitation` (reference `tasks/walk_imitation.py:19-203`, `tasks/base.py:367-428`)."""
    _MODEL, _CONTROL_TIMESTEP, _KIND, _TASK, _LOADER = 'walk', _WALK_CONTROL_TIMESTEP, st.TASK_WALK, WalkImitationTask, InferenceWalkingTrajectoryLoader
    _OBS = _WALKER_OBS + ('ref_displacement', 'ref_root_quat')

    def __init__(self, n_envs, **kw):
        super().__init__(n_envs, **kw)
        m, tg, future_steps = self.model, self.task._traj_generator, self.task._future_steps
        self._wing_spring = m.qpos_spring[self._wing_qadr]
        if self._device_bank:
            if not tg.get_joint_names():
                raise NotImplementedError('walk_imitation(device_task=True) needs a dataset that lists its mocap joints: the DeepMimic '
                                          'reward on the device compares them')
            short = [int(j) for j in np.unique(tg.traj_indices) if tg.trajectory_len(j) <= future_steps + 1]
            if short:
                raise NotImplementedError(f'trajectories {short} have at most future_steps + 1 = {future_steps + 1} rows '
                                          f'({[tg.trajectory_len(j) for j in short]}): such snippets, which the host-side task code pads '
                                          'with their last row and the reference cannot index past, are not run on the device; use '
                                          'device_task=False or leave them out of traj_indices')
        if not self._inference_mode:
            jn, sn = m.meta['jnt_names'], m.meta['site_names']
            jnames, snames = tg.get_joint_names(), tg.get_site_names()
            mj = [jn.index('walker/' + n) for n in jnames]
            self._mocap_qadr, self._mocap_vadr = m.jnt_qposadr[mj].astype(np.int64), m.jnt_dofadr[mj].astype(np.int64)
            self._mocap_sites = np.array([sn.index('walker/' + n) for n in snames], np.int64)
            self._bank = _FeatureBank()
            self._env_bank_off = np.zeros(self.n_envs, np.int64)

    def _task_obs(self, o):
        items, hidden, lists = super()._task_obs(o)
        if not self._inference_mode:                 # what get_walker_features reads (tasks/rewards.py:37-63)
            nj, ns = len(self._mocap_qadr), len(self._mocap_sites)
            hidden += [('_root_pose', 7, (7,), (st.OBS_ROOT_POSE, 0, 7)),
                       ('_root_qvel', 6, (6,), (st.OBS_QVEL, o, 6)),
                       ('_mocap_qpos', nj, (nj,), (st.OBS_QPOS, o + 6, nj)),
                       ('_mocap_qvel', nj, (nj,), (st.OBS_QVEL, o + 6 + nj, nj)),
                       ('_mocap_axes', 3 * nj, (nj, 3), (st.OBS_DOF_AXIS_EGO, o + 6 + nj, nj)),
                       ('_mocap_sites', 3 * ns, (ns, 3), (st.OBS_SITES_EGO, o + 6 + 2 * nj, ns)),
                       ('_wing_qpos', 6, (6,), (st.OBS_QPOS, o + 6 + 2 * nj + ns, 6))]
            lists += list(range(self._root_v, self._root_v + 6)) + list(self._mocap_qadr) + list(self._mocap_vadr) \
                + list(self._mocap_sites) + list(self._wing_qadr)
        return items, hidden, lists

    def _task_program(self):
        q0 = self.model.qpos0.copy()
        q0[self._wing_qadr] = self._wing_spring
        noise = self._reset_noise > 0
        return super()._task_program() | dict(reset_qpos=q0, n_noise=len(self._leg_act_qadr) if noise else 0,
                                              noise_qadr=self._leg_act_qadr if noise else None, noise_amp=self._reset_noise)

    def _bank_program(self):
        """walking: the full-body start pose and the DeepMimic reward read the bank (fb_ref_bank_wide)"""
        sl = self._obs_slices
        self._sim.ref_bank_wide(*self._bank_tables())
        return dict(randomize_start=0, start_margin=0, max_episode_rows=self.task._max_episode_steps + self.task._future_steps + 1,
                    n_mocap_joints=len(self._mocap_qadr), mocap_qadr=self._mocap_qadr, n_mocap_sites=len(self._mocap_sites),
                    obs_root_pose_off=sl['_root_pose'].start, obs_root_qvel_off=sl['_root_qvel'].start,
                    obs_mocap_qpos_off=sl['_mocap_qpos'].start, obs_mocap_qvel_off=sl['_mocap_qvel'].start,
                    obs_mocap_axes_off=sl['_mocap_axes'].start, obs_mocap_sites_off=sl['_mocap_sites'].start,
                    obs_wing_qpos_off=sl['_wing_qpos'].start, n_wing=len(self._wing_qadr), wing_qadr=self._wing_qadr,
                    wing_spring=self._wing_spring, deep_mimic_std=[rw.DEEP_MIMIC_STD[k] for k in ('com', 'qvel', 'root2site', 'joint_quat')],
                    deep_mimic_weight=_WALK_REWARD_WEIGHTS, retract_margin=_WING_RETRACT_MARGIN)

    def _snippet_root(self, snip):
        """root-joint reference (qpos [T,7], qvel [T,6]) of one loader snippet."""
        return np.asarray(snip['qpos'])[:, :7], np.asarray(snip['qvel'])[:, :6]

    def _steps_of(self, n_rows):
        t = self.task
        return min(t._max_episode_steps, n_rows - t._future_steps - 1)                               # walk_imitation.py:104-105

    def _bank_rows_of(self, j):
        """rows [T][15 + 6 nj + 3 ns] of trajectory j for fb_ref_bank_wide: root qpos, root qvel, root x, y (what a reset at the row shifts
        the root x, y by), mocap qpos, mocap qvel, root2site, joint_quat, as stored"""
        tg = self.task._traj_generator
        T = tg.trajectory_len(j)
        f = {k: np.asarray(v[:T], np.float64) for k, v in tg.full_trajectory(j).items()}
        return np.concatenate([f['root_qpos'], f['root_qvel'], f['root_qpos'][:, :2], f['qpos'], f['qvel'],
                               f['root2site'].reshape(T, -1), f['joint_quat'].reshape(T, -1)], 1)

    def _bank_tables(self):
        """... and the host mirror of the reward features (`_bank`, read by _walk_reward_factors), cut from the same fp32 rows as the
        device reads them: one block per trajectory at the trajectory's bank offset, root x, y shifted by row 0's in fp32."""
        if self._bank_rows is None:
            r = super()._bank_tables()[1]
            nj, ns = len(self._mocap_qadr), len(self._mocap_sites)
            root = r[:, :7].copy()
            root[:, :2] -= np.repeat(r[self._bank_off, 13:15], self._bank_len, 0)
            b = _FeatureBank()
            b.qpos = np.concatenate([root, r[:, 15:15 + nj]], 1).astype(np.float64)
            b.qvel = np.concatenate([r[:, 7:13], r[:, 15 + nj:15 + 2 * nj]], 1).astype(np.float64)
            b.root2site = r[:, 15 + 2 * nj:15 + 2 * nj + 3 * ns].reshape(-1, ns, 3).astype(np.float64)
            b.joint_quat = r[:, 15 + 2 * nj + 3 * ns:].reshape(-1, nj, 4).astype(np.float64)
            b._off, b._n = {j: int(o) for j, o in enumerate(self._bank_off)}, r.shape[0]
            self._bank = b
        return self._bank_len, self._bank_rows

    def _start_pose(self, ids, qpos, ref0):
        """walk_imitation.py:112-136: wings retracted (and the snippet's full-body pose, leg noise) -> qvel (None: at rest)"""
        if not self._inference_mode:          # full-body start pose from the snippet (walk_imitation.py:117-118)
            qpos[:, self._mocap_qadr] = self._bank.qpos[self._env_bank_off[ids], 7:]
        qpos[:, self._wing_qadr] = self._wing_spring
        if self._reset_noise > 0:
            qpos[:, self._leg_act_qadr] += self._rs.uniform(-self._reset_noise, self._reset_noise, (len(ids), len(self._leg_act_qadr)))
        return None

    def _task_after(self, rec, obs, resetting, time, ghost):
        """check_termination / reward / discount on the observation record of the step just taken (walk_imitation.py:152-203,
        base.py:203-225) -> step_type, reward, discount, needs_reset.  (The device-side task program `ktask_after` is the same logic;
        tests/test_device_task.py holds the two against each other.)"""
        sl = self._obs_slices
        step_now = np.round(time / self._control_timestep).astype(np.int64)
        com_dist = np.linalg.norm(obs['walker/ref_displacement'][:, 0], axis=1)
        reached_end = step_now == self._episode_steps
        linvel = np.linalg.norm(rec[:, sl['_velocimeter_now']], axis=1)
        angvel = np.linalg.norm(rec[:, sl['_gyro_now']], axis=1)
        terminate = (linvel > _TERMINAL_LINVEL) | (angvel > _TERMINAL_ANGVEL) | reached_end | \
                    (com_dist > self.task._terminal_com_dist) | self._bad_state(rec)
        if self._inference_mode:
            reward = np.ones(self.n_envs)                     # reward factors == (1,)
        else:
            reward = np.prod(self._walk_reward_factors(rec, np.minimum(step_now, self._ref_len - 1)), axis=1)
        return self._end_step(resetting, terminate, reward, time, end_ok=reached_end)

    def _walk_reward_factors(self, rec, step):
        """[N, 4 + 6]: DeepMimic factors (weights 20, 1, 1, 1) and one wing-retraction factor per wing joint
        (reference walk_imitation.py:152-177)."""
        sl = self._obs_slices
        nj, ns = len(self._mocap_qadr), len(self._mocap_sites)
        f64 = lambda k, shape=None: rec[:, sl[k]].astype(np.float64).reshape((self.n_envs,) + (shape or (-1,)))
        wf = rw.get_walker_features(f64('_root_pose'), f64('_mocap_qpos'), f64('_root_qvel'), f64('_mocap_qvel'),
                                    f64('_mocap_sites', (ns, 3)), f64('_mocap_axes', (nj, 3)))
        rows = self._env_bank_off + step
        b = self._bank
        rf = {'com': b.qpos[rows, :3], 'qvel': b.qvel[rows], 'root2site': b.root2site[rows],
              'joint_quat': np.concatenate([b.qpos[rows, None, 3:7], b.joint_quat[rows]], 1)}
        factors = rw.reward_factors_deep_mimic(wf, rf, weights=_WALK_REWARD_WEIGHTS)
        retract = linear_tolerance(f64('_wing_qpos') - self._wing_spring, _WING_RETRACT_MARGIN)
        return np.concatenate([factors, retract], 1)


class FlightImitationEnv(_ImitationEnv):
    """Batched `FlightImitationWBPG` (reference `tasks/flight_imitation.py:16-212`, `tasks/base.py:271-364`): the wing-beat pattern
    generator turns the wing actions and the beat frequency (the one user action) into ctrl."""
    _MODEL, _CONTROL_TIMESTEP, _KIND, _TASK, _LOADER = 'flight', _FLY_CONTROL_TIMESTEP, st.TASK_FLIGHT, FlightImitationTask, InferenceFlightTrajectoryLoader
    _OBS = ('accelerometer', 'actuator_activation', 'gyro', 'joints_pos', 'joints_vel', 'velocimeter', 'world_zaxis', 'ref_displacement',
            'ref_root_quat')
    _N_USER, _HOST_CTRL = 1, True

    def __init__(self, n_envs, wpg_pattern_path=None, **kw):
        super().__init__(n_envs, **kw)
        self._wbpg = BatchedWingBeatPatternGenerator(self.n_envs, base_pattern_path=wpg_pattern_path)
        self._wing_qpos_host = np.zeros((self.n_envs, 6))
        tg = self.task._traj_generator
        if self._device_bank and tg.randomize_start_step:
            short = [int(j) for j in np.unique(tg.traj_indices) if tg.trajectory_len(j) <= tg.START_MARGIN]
            if short:
                raise ValueError(f'randomize_start_step needs trajectories longer than {tg.START_MARGIN} rows; trajectories {short} have '
                                 f'{[tg.trajectory_len(j) for j in short]}')

    def _task_obs(self, o):
        items, hidden, lists = super()._task_obs(o)
        m = self.model
        return items, hidden + [('_root_pose', 7, (7,), (st.OBS_ROOT_POSE, 0, 7)),
                                ('_subtree_com', 3, (3,), (st.OBS_SUBTREE_COM, m.body_id('walker/thorax'), 3)),
                                ('_ghost_pose', 7, (7,), (st.OBS_QPOS, o, 7))], lists + list(range(self._ghost_q, self._ghost_q + 7))

    def _task_program(self):
        return super()._task_program() | self._wing_beat_program()

    def _bank_program(self):
        """flight: the draws of HDF5FlightTrajectoryLoader.get_trajectory (fb_ref_bank)"""
        tg = self.task._traj_generator
        self._sim.ref_bank(*self._bank_tables())
        return dict(randomize_start=int(bool(tg.randomize_start_step)), start_margin=tg.START_MARGIN,
                    max_episode_rows=round(self._time_limit / self._control_timestep))

    def _snippet_root(self, snip):
        com_qpos, qvel = snip                       # flight data is a CoM trajectory (flight_imitation.py:94-99)
        com_qpos = np.asarray(com_qpos)
        return np.concatenate([com2root(com_qpos[:, :3], com_qpos[:, 3:7]), com_qpos[:, 3:7]], 1), np.asarray(qvel)[:, :6]

    def _steps_of(self, n_rows):
        return min(n_rows, round(self._time_limit / self._control_timestep)) - (self.task._future_steps + 1)     # flight_imitation.py:101-106

    def _bank_rows_of(self, j):
        """rows [T][15] of trajectory j for fb_ref_bank: root qpos (com2root in fp64), CoM qvel, CoM x, y"""
        cq, cv = self.task._traj_generator.full_trajectory(j)
        cq, cv = np.asarray(cq, np.float64), np.asarray(cv, np.float64)
        return np.concatenate([com2root(cq[:, :3], cq[:, 3:7]), cq[:, 3:7], cv[:, :6], cq[:, :2]], 1)

    def _start_pose(self, ids, qpos, ref0):
        """flight_imitation.py:113-144: root linear velocity from the reference, wings on the beat pattern at a random phase -> qvel"""
        wq, wv = self._wbpg.reset(ids, self._rs.uniform(size=len(ids)))
        qpos[:, self._wing_qadr] = wq
        qvel = np.zeros((len(ids), self.model.nv))
        qvel[:, self._wing_vadr] = wv
        qvel[:, self._root_v:self._root_v + 3] = ref0[:, 7:10]
        self._wing_qpos_host[ids] = wq
        return qvel

    def _before_step(self, action, resetting):
        # wing-beat pattern at the requested frequency, as a position target turned into a force command
        wb = self._wbpg
        freq = wb.base_beat_freq * (1 + wb.rel_freq_range * action[:, -1])
        target = wb.step(freq, active=~resetting)
        action[:, self._action_indices['wings']] += target - self._wing_qpos_host
        action[np.isnan(action)] = 0.0
        return super()._before_step(self._host_ctrl(action), resetting)

    def _after_read(self, rec):
        self._wing_qpos_host = rec[:, self._obs_slices['walker/joints_pos']][:, self._wing_in_obs].astype(np.float64)

    def _before_device_step(self, resetting):
        super()._before_device_step(resetting)
        if resetting.any():                                         # the wing-beat phases the host path would draw at these resets
            ids = np.nonzero(resetting)[0]
            self._sim.task_uniforms(ids, self._rs.uniform(size=len(ids)))

    def _state_refs(self):
        return super()._state_refs() + [(self, '_wing_qpos_host'), (self._wbpg, 'freq'), (self._wbpg, 'idx'), (self._wbpg, 'pos')]

    def _task_after(self, rec, obs, resetting, time, ghost):
        """check_termination / reward / discount on the observation record of the step just taken (flight_imitation.py:170-226,
        base.py:203-225) -> step_type, reward, discount, needs_reset.  (The device-side task program `ktask_after` is the same logic;
        tests/test_device_task.py holds the two against each other.)"""
        sl = self._obs_slices
        step_now = np.round(time / self._control_timestep).astype(np.int64)
        com_dist = np.linalg.norm(obs['walker/ref_displacement'][:, 0], axis=1)
        reached_end = step_now == self._episode_steps
        height = rec[:, sl['_root_pose']][:, 2]
        terminate = (height < _TERMINAL_HEIGHT) | (com_dist > self.task._terminal_com_dist) | reached_end | self._bad_state(rec)
        # reward factors: CoM displacement and orientation error to the ghost (legs are disabled: third factor == 1)
        # (the ghost is a free body that coasts with its reference velocity during the substeps; the reference reads its
        # pose after the step, flight_imitation.py:174-176)
        ghost_com = root2com(rec[:, sl['_ghost_pose']].astype(np.float64))
        disp = np.linalg.norm(ghost_com - rec[:, sl['_subtree_com']], axis=1)
        qd = quat_dist_short_arc(np.array([1.0, 0, 0, 0]), obs['walker/ref_root_quat'][:, 0].astype(np.float64))
        reward = linear_tolerance(disp, 0.4) * linear_tolerance(qd, np.pi)
        return self._end_step(resetting, terminate, reward, time, end_ok=reached_end)


def walk_imitation(ref_path=None, force_actuators=False, disable_wings=True, traj_indices=None, random_state=None,
                   terminal_com_dist=0.3, joint_filter=0.01, n_envs=None, device=0, lib_path=None, reset_noise=0.0,
                   seed=0, max_reference_steps=None, device_task=False):
    """Batched `flybody.fly_envs.walk_imitation` (reference `fly_envs.py:100-155`).  With `ref_path` (an HDF5 walking
    dataset, or its `.npz` conversion, see `trajectory_loaders`) every env tracks its own snippet, starts from the
    snippet's full-body pose and is rewarded with the DeepMimic factors; without it the task runs in inference mode on
    the synthetic straight walk, reward 1 (`fly_envs.py:127-135`).  With `ref_path` and `device_task=True` the whole dataset is
    uploaded once as a device bank with the reward features, and every reset, the full-body start pose and the DeepMimic reward run on
    the device (`reference_picks()` reads which trajectory each env tracks).  `force_actuators`, `disable_wings=False` and `joint_filter` select
    a model variant (`flymodel.model_for`); each is tested against the oracle in tests/test_model_variants.py."""
    model = None
    if force_actuators or not disable_wings or joint_filter != 0.01:
        from .flymodel import model_for
        model = model_for('walk', force_actuators=force_actuators, use_wings=True if not disable_wings else None,
                          joint_filter=None if joint_filter == 0.01 else joint_filter)
    tg = None
    if ref_path is not None:
        tg = HDF5WalkingTrajectoryLoader(path=ref_path, random_state=random_state, traj_indices=traj_indices)
    return WalkImitationEnv(n_envs, device=device, terminal_com_dist=terminal_com_dist, time_limit=10.0,
                         future_steps=64, lib_path=lib_path, reset_noise=reset_noise, seed=seed, traj_generator=tg,
                         inference_mode=ref_path is None, max_reference_steps=max_reference_steps, device_task=device_task, model=model)


def flight_imitation(ref_path=None, wpg_pattern_path=None, force_actuators=False, disable_legs=True, traj_indices=None,
                     randomize_start_step=True, joint_filter=0.0, future_steps=5, random_state=None, terminal_com_dist=2.0,
                     n_envs=None, device=0, lib_path=None, seed=0, device_task=False):
    """Batched `flybody.fly_envs.flight_imitation` (reference `fly_envs.py:30-97`): wing-beat-pattern-generator flight
    tracking, 4 substeps of 5e-5 s per control step, 12 actions (head 3, wings 6, abdomen 2, beat frequency 1).  With
    `ref_path` every env tracks its own (randomly cut) CoM trajectory of the flight dataset; with `device_task=True` as well, the
    whole dataset is uploaded once as a device bank and every reset cuts its reference there (`reference_picks()` reads which).
    `force_actuators`, `disable_legs=False` and `joint_filter` select a model variant (`flymodel.model_for`); each is tested against the
    oracle in tests/test_model_variants.py."""
    model = None
    if force_actuators or not disable_legs or joint_filter != 0.0:      # a non-default FruitFly: compiled on first use (flymodel.model_for)
        from .flymodel import model_for
        model = model_for('flight', force_actuators=force_actuators, use_legs=True if not disable_legs else None,
                          joint_filter=None if joint_filter == 0.0 else joint_filter)
    tg = None
    if ref_path is not None:
        tg = HDF5FlightTrajectoryLoader(path=ref_path, traj_indices=traj_indices, randomize_start_step=randomize_start_step,
                                        random_state=random_state)
    return FlightImitationEnv(n_envs, device=device, terminal_com_dist=terminal_com_dist, time_limit=0.6,
                         future_steps=future_steps, lib_path=lib_path, seed=seed, wpg_pattern_path=wpg_pattern_path,
                         traj_generator=tg, device_task=device_task, model=model)


def vision_guided_flight(wpg_pattern_path=None, bumps_or_trench='bumps', force_actuators=False, disable_legs=True, random_state=None,
                         joint_filter=0.0, n_envs=None, device=0, lib_path=None, seed=0, **kwargs_arena):
    """Batched `flybody.fly_envs.vision_guided_flight` (reference `fly_envs.py:194-246`): 'bumps' or 'trench' terrain, eye
    cameras, wing-beat pattern generator, fatal ground contacts -- `flybody_b200.vision_env.BatchedVisionFlightEnv` (SURVEY.md
    8(f).1; terrain contacts against the fp64 oracle and eyes against the camera model in tests/test_hfield.py, test_eyes.py and on the
    GPU in tests/test_gpu_parity.py).  `terrain_bank=K, device_task=True` run the task's hooks on the device (FB_TASK_VISION)."""
    if force_actuators or not disable_legs or joint_filter != 0.0:
        raise NotImplementedError('only the default vision_guided_flight model variant is compiled (flybody_b200/assets/fly_vision.npz)')
    from .vision_env import BatchedVisionFlightEnv
    return BatchedVisionFlightEnv(n_envs, bumps_or_trench=bumps_or_trench, wpg_pattern_path=wpg_pattern_path, device=device, lib_path=lib_path,
                                  seed=seed, **kwargs_arena)


def template_task(random_state=None, force_actuators=False, disable_wings=True, joint_filter=0.01, adhesion_filter=0.007,
                  time_limit=1.0, mjcb_control=None, observables_options=None, action_corruptor=None, n_envs=None, device=0,
                  lib_path=None, seed=0, device_task=False):
    """Batched `flybody.fly_envs.template_task` (reference `fly_envs.py:249-300`, `tasks/template_task.py`): the walking fly
    without a ghost on flat ground, reward 1, the reference's installation test (`tests/test_core.py`) and the class to start a
    walking task from.  `force_actuators`, `disable_wings=False`, `joint_filter` and `adhesion_filter` select a model variant
    (`flymodel.model_for('template', ...)`).  `device_task=True` runs the task hooks on the device (FB_TASK_TEMPLATE), which `step_device` needs.
    `mjcb_control` (a per-substep Python callback) and `observables_options` are not supported."""
    if mjcb_control is not None:
        raise NotImplementedError('mjcb_control: a per-substep Python callback cannot run at batch speed (DESIGN.md section 8). Perturbation '
                                  'forces go through env.set_applied_forces(qfrc=..., xfrc=...), the batched physics.data.qfrc_applied / '
                                  'xfrc_applied, which act in every substep until overwritten')
    if observables_options is not None:
        raise NotImplementedError('observables_options (observable noise, delay, buffering) are not supported')
    model = None
    if force_actuators or not disable_wings or joint_filter != 0.01 or adhesion_filter != 0.007:
        from .flymodel import model_for
        model = model_for('template', force_actuators=force_actuators, use_wings=True if not disable_wings else None,
                          joint_filter=None if joint_filter == 0.01 else joint_filter,
                          adhesion_filter=None if adhesion_filter == 0.007 else adhesion_filter)
    return TemplateTaskEnv(n_envs, time_limit=time_limit, action_corruptor=action_corruptor, random_state=random_state, device=device,
                           lib_path=lib_path, seed=seed, device_task=device_task, model=model)


def walk_on_ball(force_actuators=False, disable_wings=True, random_state=None, n_envs=None, device=0, lib_path=None, seed=0,
                 device_task=False):
    """Batched `flybody.fly_envs.walk_on_ball` (reference `fly_envs.py:158-191`, `tasks/walk_on_ball.py`): the tethered fly walking on
    a floating ball, 10 substeps of 2e-4 s per control step, a 2 s time limit, 59 actions and the ten walker observables plus
    `walker/ball_qvel`.  `force_actuators` and `disable_wings=False` select a model variant (`flymodel.model_for('ball', ...)`).
    `device_task=True` runs the task hooks on the device (FB_TASK_BALL), which `step_device` needs."""
    model = None
    if force_actuators or not disable_wings:
        from .flymodel import model_for
        model = model_for('ball', force_actuators=force_actuators, use_wings=True if not disable_wings else None)
    return WalkOnBallEnv(n_envs, random_state=random_state, device=device, lib_path=lib_path, seed=seed, device_task=device_task,
                         model=model)

