"""Batched `flybody.fly_envs.vision_guided_flight` (reference `fly_envs.py:194-246`, `tasks/vision_flight.py`,
`tasks/base.py:271-364`, `tasks/arenas/hills.py`): flight over a per-episode heightfield terrain ('bumps' or 'trench') with
a controllable wing-beat pattern generator, egocentric eye cameras, fatal ground contacts.

SURVEY.md 8(f).1, verified under host emulation and on the GPU (tests/test_gpu_parity.py): the physics
is the `vision` model variant (flight model without a ghost, ground contacts on, terrain geom), terrain contacts come from the
heightfield narrowphase (`fb_hfield_collision`, MuJoCo's prism walk + MPR, restated from memory), the eyes from the device ray
caster (`fb_render_eyes`: MuJoCo's camera model, not its OpenGL image).  The task logic -- episode initialisation, the
wing-beat generator in `before_step`, the seven reward factors, termination -- mirrors the reference in vectorised numpy on
the read-back record, in the host control step every env shares (`fly_envs._TaskEnv`).
"""
import collections

import numpy as np

from . import arenas
from . import stepper as st
from .dm_env_shim import Array
from .fly_envs import BatchedWingBeatPatternGenerator, _TaskEnv, _device_tensor, _pinned
from .flymodel import load_model
from .synthetic import _FLY_CONTROL_TIMESTEP

_BODY_PITCH_ANGLE = 47.5          # reference tasks/constants.py: body pitch of the hover pose, degrees


def _tolerance_linear(x, lo, hi, margin):
    """`dm_control.utils.rewards.tolerance(x, bounds=(lo, hi), sigmoid='linear', margin, value_at_margin=0)`."""
    x = np.asarray(x, np.float64)
    d = np.where(x < lo, lo - x, np.where(x > hi, x - hi, 0.0)) / margin
    return np.where(d <= 0, 1.0, np.clip(1.0 - d, 0.0, 1.0))


class BatchedVisionFlightEnv(_TaskEnv):
    """dm_env-shaped environment over N lock-stepped flies on their own terrains."""
    # head 3, wings 6, abdomen 2 actions + 1 user action (beat frequency); the wing-beat generator builds ctrl on the host
    _CONTROL_TIMESTEP, _KIND, _N_USER, _HOST_CTRL = _FLY_CONTROL_TIMESTEP, st.TASK_VISION, 1, True
    _OBS = ('accelerometer', 'actuator_activation', 'gyro', 'joints_pos', 'joints_vel', 'left_eye', 'right_eye', 'velocimeter', 'world_zaxis',
            'task_input')

    def __init__(self, n_envs, bumps_or_trench='bumps', wpg_pattern_path=None, device=0, lib_path=None, seed=0, eye_camera_size=32,
                 eye_camera_fovy=150.0, target_height_range=(0.5, 0.8), target_speed_range=(20, 40), init_pos_x_range=(-5, -5),
                 init_pos_y_range=(0, 0), time_limit=0.4, floor_contacts_fatal=True, terrain_bank=None, device_task=False, **kwargs_arena):
        if bumps_or_trench not in ('bumps', 'trench'):
            raise ValueError("Only 'bumps' and 'trench' terrains are supported.")
        super().__init__(load_model('vision'), n_envs, device, lib_path, time_limit, seed, device_task)
        m, N = self.model, self.n_envs
        self._fatal = floor_contacts_fatal
        self._wbpg = BatchedWingBeatPatternGenerator(N, base_pattern_path=wpg_pattern_path)
        cls = arenas.SineBumps if bumps_or_trench == 'bumps' else arenas.SineTrench
        self._arenas = [cls(**kwargs_arena) for _ in range(N)]
        a0 = self._arenas[0]
        assert (a0.nrow, a0.ncol) == (m.meta['hf_nrow'], m.meta['hf_ncol']) and a0.size[0] == m.hf_size[0], 'arena grid differs from the compiled model'
        self._half = float(a0.size[0])
        self._terrain = np.zeros((N, a0.nrow, a0.ncol), np.float32)
        # The reference draws a new terrain every episode (16 ms of scipy per terrain here).  `terrain_bank=K` pre-generates K
        # terrains and lets every episode pick one at random instead -- the same distribution over a finite bank, for large batches.
        self._bank = None
        if terrain_bank:
            self._bank = []
            for _ in range(int(terrain_bank)):
                t = a0.generate(self._rs)
                self._bank.append((t.astype(np.float32), a0.trench_specs))
        self._sim.hfield_collision(m.meta['hf_geom'], m.hf_size, a0.nrow, a0.ncol, m.hf_pair_geom)
        self._ranges = dict(h=target_height_range, v=target_speed_range, x=init_pos_x_range, y=init_pos_y_range)
        sens = m.meta['sensor_names']
        sd = lambda n: int(m.sensor_adr[sens.index('walker/' + n)])
        up = m.site_quat[m.meta['site_names'].index('walker/hover_up_dir')].copy()
        up[0] *= -1.0                                        # neg_quat(up_dir): the hover pose (vision_flight.py:124-126)
        self._hover_quat = up
        th = np.deg2rad(_BODY_PITCH_ANGLE)
        self._target_zaxis = np.array([np.sin(th), 0.0, np.cos(th)])
        # observation program (device): the walker observables + what reward / termination read
        nq = len(self._obs_qadr)
        rows = [('walker/accelerometer', 3, (st.OBS_SENSOR_MEAN, sd('accelerometer'), 3)), ('walker/gyro', 3, (st.OBS_SENSOR_MEAN, sd('gyro'), 3)),
                ('walker/joints_pos', nq, (st.OBS_QPOS, 0, nq)), ('walker/joints_vel', nq, (st.OBS_QVEL, nq, nq)),
                ('walker/velocimeter', 3, (st.OBS_SENSOR_MEAN, sd('velocimeter'), 3)), ('walker/world_zaxis', 3, (st.OBS_ROOT_ZAXIS, 0, 3)),
                ('_velocimeter_now', 3, (st.OBS_SENSOR_NOW, sd('velocimeter'), 3)), ('_root_pose', 7, (st.OBS_ROOT_POSE, 0, 7)),
                ('_root_qvel', 6, (st.OBS_QVEL, 2 * nq, 6)), ('_scalars', 3, (st.OBS_SCALARS, 0, 3)),
                ('_world_contact', 1, (st.OBS_WORLD_CONTACT, 0, 1)), ('_task_target', 2, (st.OBS_TASK_TARGET, 0, 2))]
        self._upload_obs_program([(n, w, (w,), item) for n, w, item in rows],
                                 list(self._obs_qadr) + list(self._obs_vadr) + list(range(self._root_v, self._root_v + 6)))
        self._sl = self._obs_slices
        # eyes
        self._eye_program(eye_camera_size, eye_camera_fovy, a0.nrow, a0.ncol, self._half, float(m.geom_pos[m.meta['hf_geom']][2]))
        self._eye_size = eye_camera_size
        self._eyes_host = _pinned((N, 2, eye_camera_size, eye_camera_size, 3), np.uint8)      # D2H target of every step's render
        # per-env episode state
        self._target_height, self._target_speed = np.zeros(N), np.zeros(N)
        self._wing_qpos = np.zeros((N, 6))
        self._has_trench = np.zeros(N, bool)
        self._last_draws = np.zeros((N, 8), np.float32)
        # task hooks on the device (fb_task_*, FB_TASK_VISION): needs the terrain bank (a resetting env copies one of its terrains on the device)
        if self._device_task:
            if self._bank is None:
                raise NotImplementedError('device_task=True needs terrain_bank=K (a resetting env copies one of the K terrains on the device)')
            self._upload_task_program(seed)

    def eyes_device(self):
        """zero-copy torch view [n_envs, 2, size, size, 3] uint8 (index 0 right eye, 1 left eye) of the images the last step rendered,
        on this env's device -- for a policy that lives on the GPU (the numpy observation holds the same images on the host)."""
        if self._eyes_dev is None:
            ptr, nbytes = self._sim.eyes_ptr()
            self._eyes_dev = _device_tensor(ptr, (self.n_envs, 2, self._eye_size, self._eye_size, 3), '|u1', self._sim.device)
        return self._eyes_dev

    # ---------------------------------------------------------------------------------- specs
    def observation_spec(self):
        lead = (self.n_envs,) if self._batched else ()
        nq, s = len(self._obs_qadr), self._eye_size
        shapes = {'accelerometer': (3,), 'actuator_activation': (0,), 'gyro': (3,), 'joints_pos': (nq,), 'joints_vel': (nq,), 'left_eye': (s, s, 3),
                  'right_eye': (s, s, 3), 'velocimeter': (3,), 'world_zaxis': (3,), 'task_input': (2,)}
        return collections.OrderedDict(('walker/' + k, Array(lead + shapes[k], np.uint8 if 'eye' in k else np.float32, name='walker/' + k)) for k in self._OBS)

    @property
    def target_height(self):
        return self._target_height.copy()

    @property
    def target_speed(self):
        return self._target_speed.copy()

    def _upload_task_program(self, seed):
        """fb_task_program FB_TASK_VISION: the hooks of this env as a device-side program (same constants as the host path); `seed`
        seeds the device's counter-hash draws."""
        self._seed = seed
        r = self._ranges
        self._sim.hfield_bank(np.stack([t for t, _ in self._bank]))
        dummy = np.zeros((1, 7), np.float32); dummy[0, 3] = 1.0
        trench = {}
        if self._bank[0][1] is not None:                                 # 'trench' arenas: the corridor's centre line of every bank terrain
            cap = max(len(sp['y_coords']) for _, sp in self._bank)
            ty = np.zeros((len(self._bank), cap), np.float32)
            for k, (_, sp) in enumerate(self._bank):
                ty[k, :len(sp['y_coords'])] = sp['y_coords']
            trench = dict(trench_cap=cap, trench_y=ty, trench_len=np.array([len(sp['y_coords']) for _, sp in self._bank], np.int32),
                          trench_x=np.array([[sp['x_coords'][0], sp['x_coords'][-1]] for _, sp in self._bank], np.float32))
        self._sim.task_program(**self._task_program() | self._wing_beat_program() | dict(
            episode_steps=1 << 30, ref_len=1, ref_qpos=dummy, ref_qvel=np.zeros((1, 6), np.float32), target_height_range=r['h'],
            target_speed_range=r['v'], init_x_range=r['x'], init_y_range=r['y'], hover_quat=self._hover_quat, target_zaxis=self._target_zaxis,
            floor_contacts_fatal=1 if self._fatal else 0, **trench))
        self._dev_views = None

    def _state_refs(self):
        return super()._state_refs() + [(self, '_target_height'), (self, '_target_speed')]

    def _state_prepare(self):
        if not self._device_task:
            raise NotImplementedError('state rows do not cover the host-side vision task (per-env terrains and draws live on the host): '
                                      'use terrain_bank=K, device_task=True')

    def _before_device_step(self, resetting):
        draws = getattr(self, '_forced_draws', None)               # (tests: the draws the host-side code would make at these resets)
        if draws is not None and resetting.any():
            ids = np.nonzero(resetting)[0]
            self._sim.task_uniform_rows(ids, draws[ids])

    def _after_device_step(self, resetting):
        tgt = self._rec[:, self._sl['_task_target']]
        self._target_height, self._target_speed = tgt[:, 0].astype(np.float64), tgt[:, 1].astype(np.float64)

    def step_device(self, action):
        """Device-resident control step (see `_TaskEnv.step_device`): `action` a CUDA tensor [n_envs, 12]; returns zero-copy torch
        views (observation rows, out [n_envs, 4] = reward, discount, step_type, 0, eyes uint8 [n_envs, 2, S, S, 3]); nothing is copied to
        the host and the call does not synchronise.  Column slices of the rows: `observation_layout()`."""
        views = super().step_device(action)
        self._sim.render_eyes_async()
        return views + (self.eyes_device(),)

    def observation_layout(self):
        """{observable name: column slice} of the observation rows `step_device` returns (eyes come as their own tensor)"""
        sl = self._sl
        return {k: v for k, v in sl.items() if not k.startswith('_')} | {'walker/task_input': sl['_task_target']}

    def hfield_height(self, x, y):
        """`VisionFlightImitationWBPG.get_hfield_height` per env: height at the grid point nearest to (x, y)."""
        return arenas.hfield_height(self._terrain, x, y, self._half)

    # -------------------------------------------------------------------------------- episode
    def _reset_envs(self, ids, hold=False):
        """initialize_episode_mjcf + initialize_episode (vision_flight.py:97-139): targets, start point, wing-beat phase, a new
        terrain (hills.py:442-473 / 333-392), the fly in its hover pose `target_height` above the terrain at the target speed."""
        m, r = self.model, self._ranges
        n = len(ids)
        qpos, qvel = np.tile(m.qpos0, (n, 1)), np.zeros((n, m.nv))
        for k, e in enumerate(ids):
            # one row of six uniforms per episode, in the order the device-side task program consumes them (fb_task_uniform_rows):
            # target height, target speed, start x, start y, wing-beat phase, terrain pick
            u = self._rs.uniform(size=6)
            self._last_draws[e, :6] = u
            self._target_height[e] = r['h'][0] + (r['h'][1] - r['h'][0]) * u[0]
            self._target_speed[e] = r['v'][0] + (r['v'][1] - r['v'][0]) * u[1]
            x, y = r['x'][0] + (r['x'][1] - r['x'][0]) * u[2], r['y'][0] + (r['y'][1] - r['y'][0]) * u[3]
            wq, _ = self._wbpg.reset(np.array([e]), np.array([u[4]]))
            if self._bank is None:
                self._terrain[e] = self._arenas[e].generate(self._rs)
            else:
                self._terrain[e], self._arenas[e].trench_specs = self._bank[min(int(u[5] * len(self._bank)), len(self._bank) - 1)]
            self._has_trench[e] = self._arenas[e].trench_specs is not None
            z = float(arenas.hfield_height(self._terrain[e], [x], [y], self._half)[0]) + self._target_height[e]
            qpos[k, self._root_q:self._root_q + 3] = (x, y, z)
            qpos[k, self._root_q + 3:self._root_q + 7] = self._hover_quat
            qpos[k, self._wing_qadr] = wq[0]
            qvel[k, self._root_v] = self._target_speed[e]
            self._wing_qpos[e] = wq[0]
        self._sim.hfield_write(ids, self._terrain[ids])
        self._start_episodes(ids, qpos, qvel, hold)

    def _before_step(self, action, resetting):
        # before_step (vision_flight.py:141-155): wing-beat pattern at the requested frequency, position target -> force command
        action[np.isnan(action)] = 0.0
        wb = self._wbpg
        target = wb.step(wb.base_beat_freq * (1 + wb.rel_freq_range * action[:, -1]), active=~resetting)
        action[:, self._action_indices['wings']] += np.where(resetting[:, None], 0.0, target - self._wing_qpos)
        ctrl = self._host_ctrl(action)
        return ctrl, ctrl.nbytes

    def _after_read(self, rec):
        self._wing_qpos = rec[:, self._sl['walker/joints_pos']][:, self._wing_in_obs].astype(np.float64)

    def _observation(self, rec):
        sl, N = self._sl, self.n_envs
        eyes = self._sim.render_eyes(self._eyes_host)
        obs = collections.OrderedDict()
        for k in self._OBS:
            name = 'walker/' + k
            if k == 'actuator_activation':
                obs[name] = np.zeros((N, 0), np.float32)
            elif k == 'left_eye':
                obs[name] = eyes[:, 1]
            elif k == 'right_eye':
                obs[name] = eyes[:, 0]
            elif k == 'task_input':
                obs[name] = np.stack([self._target_height, self._target_speed], 1).astype(np.float32)
            else:
                obs[name] = rec[:, sl[name]]
        return obs

    def _task_after(self, rec, obs, resetting, time, ghost):
        """get_reward (vision_flight.py:157-233), check_termination (a bad state, base.py:222-225, or a fatal floor contact), get_discount;
        the device task FB_TASK_VISION is the same logic"""
        reward = np.prod(self.reward_factors(rec), axis=1)
        terminate = self._bad_state(rec) | (self.floor_contact() if self._fatal else False)
        return self._end_step(resetting, terminate, reward, time)

    # -------------------------------------------------------------------------- task quantities
    def floor_contact(self):
        """`check_floor_contact` (vision_flight.py:235-247): an active contact (efc_address >= 0) with a geom of the world body (ground
        plane, terrain) -- evaluated on the device by the observation program (FB_OBS_WORLD_CONTACT), read from the record."""
        return self._rec[:, self._sl['_world_contact']][:, 0] > 0.5

    def reward_factors(self, rec):
        """[N, 6] (vision_flight.py:157-233): height above the terrain, forward speed, speed, side speed, body axis, centre of
        the trench; the leg-retraction factor is empty with disabled legs."""
        sl = self._sl
        pose, vel = rec[:, sl['_root_pose']].astype(np.float64), rec[:, sl['_root_qvel']].astype(np.float64)[:, :3]
        ts, th = self._target_speed, self._target_height
        height = _tolerance_linear(pose[:, 2] - self.hfield_height(pose[:, 0], pose[:, 1]), th, th, 0.15)
        x_speed = _tolerance_linear(vel[:, 0], ts, np.inf, 1.1 * ts)
        speed = _tolerance_linear(np.linalg.norm(vel, axis=1), ts, ts, 1.1 * ts)
        side = _tolerance_linear(rec[:, sl['_velocimeter_now']][:, 1], 0.0, 0.0, 10.0)
        zaxis = rec[:, sl['walker/world_zaxis']].astype(np.float64)
        ang = np.arccos(np.clip(zaxis @ self._target_zaxis, -1.0, 1.0))
        world_zaxis = _tolerance_linear(ang, 0.0, 0.0, np.pi)
        centre = np.ones(self.n_envs)
        for e in np.nonzero(self._has_trench)[0]:                       # ('bumps' arenas have no trench: nothing to do)
            spec = self._arenas[e].trench_specs
            if spec['x_coords'][0] <= pose[e, 0] <= spec['x_coords'][-1]:
                yc = spec['y_coords'][np.abs(spec['x_coords'] - pose[e, 0]).argmin()]
                centre[e] = _tolerance_linear(pose[e, 1], yc, yc, 0.15)
        return np.stack([height, x_speed, speed, side, world_zaxis, centre], 1)
