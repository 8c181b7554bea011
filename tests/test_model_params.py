"""Per-env model parameters (fb_param_*): the step with an env's overlay row equals a handle created from a model patched with the same raw
fields, bit for bit, and holds the fp64 oracle of that model to the parity tolerances; known answers; the null path; persistence; state
rows; draws at resets on the host-side and the device-side task code; the queries; input checks.  CPU tier: the host-emulation build of
the kernel source.  GPU tier (-m gpu): the same on the H100 at 4096 envs."""
import numpy as np
import pytest

import __graft_entry__ as ge
from flybody_b200 import fly_envs
from flybody_b200 import stepper as st
from flybody_b200.flymodel import load_model
from parity_common import compare_stage_fields, random_state, summarize_tf, teacher_forced_errors

FIELD = {'body_mass': 'body_mass', 'body_inertia': 'body_inertia', 'dof_armature': 'dof_armature', 'dof_damping': 'dof_damping',
         'jnt_stiffness': 'jnt_stiffness', 'geom_friction': 'geom_friction', 'actuator_gainprm': 'actuator_gainprm',
         'actuator_biasprm': 'actuator_biasprm', 'gravity': 'opt_gravity', 'wind': 'opt_wind', 'density': 'opt_density',
         'viscosity': 'opt_viscosity'}
OUTPUTS = (st.QPOS, st.QVEL, st.ACT, st.SENSORDATA, st.EFC_FORCE)


@pytest.fixture(scope='module')
def emu():
    ge.build()
    return ge.EMU


def nominal(m, name):
    return np.asarray(m.a[FIELD[name]], np.float64).reshape(-1)


def random_params(m, seed):
    """every parameter within +-30 % of its nominal value (wind, nominal 0: up to 10 cm/s), rounded to fp32"""
    rs = np.random.RandomState(seed)
    out = {}
    for name in st.PARAMS:
        v = nominal(m, name)
        v = rs.uniform(-10, 10, 3) if name == 'wind' else v * rs.uniform(0.7, 1.3, v.shape)
        out[name] = v.astype(np.float32)
    return out


def patched(m, params):
    """FlyModel.copy() with the raw fields replaced; the derived ones stay as compiled"""
    p = m.copy()
    for name, v in params.items():
        p.a[FIELD[name]] = np.asarray(v, np.float64).reshape(np.shape(m.a[FIELD[name]]))
    return p.rebuild()


def start_state(m, seed):
    """the model's reset pose (template: contacts at qpos0) with random joint velocities; flight: lifted 2 cm into the air"""
    q, v = random_state(m, seed, 0.05, 0.5)
    if m.nu != 59:
        q[int(m.jnt_qposadr[0]) + 2] += 2.0
    return q, v


def run(sim, q, v, ctrl, steps=3, n_sub=None):
    sim.reset(q, v)
    sim.set_control(ctrl)
    for _ in range(steps):
        sim.step(n_sub or 5)
    obs = sim.read_obs()
    sim.forward()                                           # the constraint forces of the current rows (the step's are of its last substep)
    out = [sim.get(f) for f in OUTPUTS] + [obs]
    nefc = sim.get(st.NEFC)[:, 0].astype(np.int64)
    out[OUTPUTS.index(st.EFC_FORCE)][np.arange(st.MAXEFC)[None] >= nefc[:, None]] = 0      # (rows past nefc are not outputs)
    return out


def equal_rows(a, b):
    for x, y in zip(a, b):
        assert np.array_equal(x.view(np.uint32), y.view(np.uint32))


@pytest.mark.parametrize('variant', ['template', 'flight'])
def test_overlay_steps_like_a_patched_model_bit_for_bit(emu, variant):
    m = load_model(variant)
    n = 3
    params = [random_params(m, 10 * k + 1) for k in range(n)]
    sim = st.BatchedStepper(m, n, lib_path=emu)
    for name in st.PARAMS:
        sim.param_set(name, np.stack([p[name] for p in params]))
    for name in st.PARAMS:
        assert np.array_equal(sim.param_get(name), np.stack([p[name] for p in params]))
    q, v = start_state(m, 4)
    ctrl = np.random.RandomState(5).uniform(-0.5, 0.5, (n, m.nu))
    got = run(sim, q, v, ctrl)
    for k in range(n):
        one = st.BatchedStepper(patched(m, params[k]), 1, lib_path=emu)
        ref = run(one, q, v, ctrl[k:k + 1])
        for x, y in zip(got, ref):
            assert np.array_equal(x[k:k + 1].view(np.uint32), y.view(np.uint32)), (variant, k)
    if variant == 'template':
        assert sim.get(st.NCON)[:, 0].min() > 0                 # the contacts (and their friction) took part


@pytest.mark.parametrize('variant', ['template', 'flight'])
def test_overlay_env_matches_the_oracle_of_its_patched_model(emu, variant):
    m = load_model(variant)
    params = random_params(m, 7)
    mp = patched(m, params)
    sim = st.BatchedStepper(m, 2, lib_path=emu)
    for name, v in params.items():
        sim.param_set(name, v, env_ids=[0])
    compare_stage_fields(mp, sim, seed=3, env=0, act=True)
    # the gates of test_model_variants.test_teacher_forced_control_steps, with its control steps (walk 10 substeps, flight 4 with
    # smaller actions)
    tf = dict(n_sub=10) if variant == 'template' else dict(n_sub=4, ctrl_scale=0.2)
    r = summarize_tf(*teacher_forced_errors(mp, sim, 20, **tf))
    assert r['p90_q'] < 2e-6 and r['p90_v'] < 2e-3 and r['hist_v']['<0.005'] >= 18 and r['p90_s'] < 1e-3, r


def test_no_gravity_no_fluid_keeps_the_linear_momentum(emu):
    """zero gravity, density and viscosity on the flight model in the air: every force left is internal (joints, actuators, self-
    contacts), so the rate of the fly's linear momentum, the root's translational rows of M qacc + qfrc_bias, is 0 to fp32 rounding"""
    m = load_model('flight')
    sim = st.BatchedStepper(m, 2, lib_path=emu)
    for name in ('gravity', 'density', 'viscosity'):
        sim.param_set(name, np.zeros_like(nominal(m, name)), env_ids=[1])
    q, v = start_state(m, 2)
    rv, mass = int(m.jnt_dofadr[0]), float(m.body_subtreemass[1])
    sim.reset(q, v)
    sim.set_control(np.random.RandomState(1).uniform(-0.5, 0.5, (2, m.nu)))
    for k in range(3):
        sim.step(4)
        sim.forward()
        con = sim.get(st.CONTACT).reshape(2, st.MAXCON, 16)
        g12 = con[1, :int(sim.get(st.NCON)[1, 0]), 7:9].astype(np.int64)
        assert not (m.geom_bodyid[g12] == 0).any(), g12
        M = sim.get(st.QM_DENSE).reshape(2, m.nv, m.nv).astype(np.float64)
        a_com = (np.einsum('eij,ej->ei', M[:, rv:rv + 3], sim.get(st.QACC).astype(np.float64)) + sim.get(st.QFRC_BIAS)[:, rv:rv + 3]) / mass
        assert np.abs(a_com[1]).max() < 1e-4 * 981, a_com[1]


def test_scaled_gain_and_bias_scale_the_actuator_force(emu):
    m = load_model('flight')
    sim = st.BatchedStepper(m, 2, lib_path=emu)
    s = np.array([[1.0], [2.0]], np.float32)
    sim.param_set('actuator_gainprm', nominal(m, 'actuator_gainprm')[None] * s)
    sim.param_set('actuator_biasprm', nominal(m, 'actuator_biasprm')[None] * s)
    q, v = start_state(m, 6)
    sim.reset(q, v)
    sim.set_control(np.random.RandomState(2).uniform(-0.8, 0.8, m.nu))
    sim.forward()
    f = sim.get(st.QFRC_ACTUATOR)
    dofs = [int(m.jnt_dofadr[m.actuator_trnid[i]]) for i in range(m.nu) if m.actuator_trntype[i] == 0 and not m.actuator_forcelimited[i]]
    assert len(dofs) >= 5 and np.abs(f[0, dofs]).min() > 0
    assert np.array_equal(f[1, dofs], 2 * f[0, dofs])


def test_null_path_compiled_values_clear_and_other_envs(emu):
    m = load_model('template')
    n = 3
    q, v = start_state(m, 8)
    ctrl = np.random.RandomState(9).uniform(-0.5, 0.5, (n, m.nu))
    ref = run(st.BatchedStepper(m, n, lib_path=emu), q, v, ctrl)
    sim = st.BatchedStepper(m, n, lib_path=emu)
    for name in st.PARAMS:                                  # unset: the compiled values
        assert np.array_equal(sim.param_get(name), np.tile(nominal(m, name).astype(np.float32), (n, 1)))
    sim.param_set('body_mass', nominal(m, 'body_mass'))    # an overlay at the compiled values
    for name in st.PARAMS:
        sim.param_set(name, nominal(m, name))
    equal_rows(run(sim, q, v, ctrl), ref)
    p = random_params(m, 3)
    for name in st.PARAMS:                                  # env 1 only: the other envs keep their bits
        sim.param_set(name, p[name], env_ids=[1])
    got = run(sim, q, v, ctrl)
    for e in (0, 2):
        equal_rows([x[e:e + 1] for x in got], [x[e:e + 1] for x in ref])
    assert not np.array_equal(got[0][1], ref[0][1])
    sim.param_clear()
    for name in st.PARAMS:
        assert np.array_equal(sim.param_get(name), np.tile(nominal(m, name).astype(np.float32), (n, 1)))
    equal_rows(run(sim, q, v, ctrl), ref)


def test_values_persist_across_steps_and_resets(emu):
    m = load_model('template')
    sim = st.BatchedStepper(m, 3, lib_path=emu)
    p = random_params(m, 4)
    sim.param_set('dof_damping', p['dof_damping'], env_ids=[2])
    sim.param_set('gravity', [0.0, 0.0, -500.0])
    q, v = start_state(m, 1)
    sim.reset(q, v); sim.step(5); sim.reset(q, v, env_ids=[2]); sim.reset_hold([1], q); sim.step(5)
    assert np.array_equal(sim.param_get('dof_damping')[2], p['dof_damping'])
    assert np.array_equal(sim.param_get('dof_damping')[0], nominal(m, 'dof_damping').astype(np.float32))
    assert np.all(sim.param_get('gravity') == np.float32([0, 0, -500]))


def test_state_rows_carry_the_parameters(emu):
    m = load_model('template')
    n = 3
    sim = st.BatchedStepper(m, n, lib_path=emu)
    sim.state_bank(4)
    sim.save_state(slots=[0], env_ids=[0])
    slots0 = sim.state_slots
    p = random_params(m, 5)
    for name in st.PARAMS:
        sim.param_set(name, p[name], env_ids=[0])
    with pytest.raises(st.StepperError, match='dropped'):   # the overlay changed the row layout
        sim.save_state(slots=[0], env_ids=[0])
    assert sim.state_slots > slots0
    sim.state_bank(4)
    q, v = start_state(m, 2)
    sim.reset(q, v)
    sim.set_control(np.random.RandomState(3).uniform(-0.5, 0.5, (n, m.nu)))
    sim.step(5)
    sim.save_state(slots=[1], env_ids=[0])
    sim.step(5)
    cont = [sim.get(f)[0:1] for f in OUTPUTS[:-1]]
    sim.load_state(slots=[1], env_ids=[2])                  # env 0's row into env 2: its parameters come along
    assert np.array_equal(sim.param_get('body_mass')[2], p['body_mass'])
    sim.step(5)
    equal_rows([sim.get(f)[2:3] for f in OUTPUTS[:-1]], cont)
    sim.param_clear()
    with pytest.raises(st.StepperError, match='dropped'):
        sim.load_state(slots=[1], env_ids=[2])


def test_draws_at_resets(emu):
    m = load_model('template')
    n = 4
    lo = {'body_mass': nominal(m, 'body_mass') * 0.8, 'geom_friction': nominal(m, 'geom_friction') * 0.5}
    hi = {'body_mass': nominal(m, 'body_mass') * 1.2, 'geom_friction': nominal(m, 'geom_friction') * 1.5}
    q, _ = start_state(m, 1)

    def fresh(seed):
        sim = st.BatchedStepper(m, n, lib_path=emu)
        sim.param_draws('body_mass', lo['body_mass'], hi['body_mass'], shared=True, seed=seed)
        sim.param_draws('geom_friction', lo['geom_friction'], hi['geom_friction'], seed=seed)
        return sim
    sim = fresh(11)
    assert np.array_equal(sim.param_get('body_mass'), np.tile(nominal(m, 'body_mass').astype(np.float32), (n, 1)))   # no reset yet
    rows = []
    for k in range(3):
        sim.reset(q)
        r = {name: sim.param_get(name) for name in lo}
        sim.set_control(np.zeros(m.nu)); sim.step(3)
        for name in lo:                                     # unchanged by steps
            assert np.array_equal(sim.param_get(name), r[name])
        rows.append(r)
    for r in rows:
        for name in lo:
            assert np.all(r[name] >= lo[name].astype(np.float32)) and np.all(r[name] <= hi[name].astype(np.float32))
        with np.errstate(invalid='ignore'):
            f = r['body_mass'] / nominal(m, 'body_mass')[None]
        f = f[:, nominal(m, 'body_mass') > 0]
        assert np.allclose(f, f[:, :1], rtol=1e-6)           # shared: one factor per env
        assert len(np.unique(np.round(f[:, 0], 6))) == n      # ... of its own
        g = r['geom_friction'] / np.where(nominal(m, 'geom_friction') > 0, nominal(m, 'geom_friction'), 1)[None]
        assert np.std(g[0, nominal(m, 'geom_friction') > 0]) > 0.05    # per element
    assert not np.array_equal(rows[0]['body_mass'], rows[1]['body_mass'])
    sim.reset(q, env_ids=[2])                               # a partial reset draws the listed env only
    r = sim.param_get('body_mass')
    assert np.array_equal(r[[0, 1, 3]], rows[2]['body_mass'][[0, 1, 3]]) and not np.array_equal(r[2], rows[2]['body_mass'][2])
    again = fresh(11)                                       # the same seed and reset sequence: the same rows
    for k in range(3):
        again.reset(q)
    assert np.array_equal(again.param_get('geom_friction'), rows[2]['geom_friction'])
    other = fresh(12)
    other.reset(q)
    assert not np.array_equal(other.param_get('geom_friction'), rows[0]['geom_friction'])
    sim.param_draws('body_mass')                            # stop drawing one parameter
    sim.reset(q)
    assert np.array_equal(sim.param_get('body_mass'), r) and not np.array_equal(sim.param_get('geom_friction'), rows[2]['geom_friction'])


def drive_envs(env, actions):
    env.reset()
    rows = []
    for a in actions:
        env.step(a)
        rows.append(env.model_params())
    return rows


def test_host_and_device_task_code_draw_the_same_rows(emu):
    n = 3
    rs = np.random.RandomState(0)
    actions = rs.uniform(-0.5, 0.5, (24, n, 59)).astype(np.float32)
    out = []
    for device_task in (False, True):
        env = fly_envs.template_task(n_envs=n, lib_path=emu, device_task=device_task, time_limit=0.02)      # LAST every 10 steps
        m = env.model
        env.randomize_model_params(seed=5, shared=('body_mass',), body_mass=(nominal(m, 'body_mass') * 0.9, nominal(m, 'body_mass') * 1.1),
                                   dof_damping=(nominal(m, 'dof_damping') * 0.7, nominal(m, 'dof_damping') * 1.3),
                                   gravity=([0, 0, -1000.0], [0, 0, -960.0]))
        out.append(drive_envs(env, actions))
        env.close()
    host, dev = out
    for a, b in zip(host, dev):
        for name in st.PARAMS:
            assert np.array_equal(a[name], b[name]), name
    assert not np.array_equal(host[0]['dof_damping'], host[-1]['dof_damping'])      # the auto-resets drew again


def test_queries_with_parameters(emu):
    m = load_model('template')
    n = 2
    p = random_params(m, 6)
    sim = st.BatchedStepper(m, n, lib_path=emu)
    for name in st.PARAMS:
        sim.param_set(name, p[name], env_ids=[1])
    one = st.BatchedStepper(patched(m, p), 1, lib_path=emu)
    q, v = start_state(m, 3)
    qacc = np.random.RandomState(4).uniform(-100, 100, (n, m.nv))
    for s in (sim, one):
        s.reset(q, v)
    sim.inverse(qacc)
    one.inverse(qacc[1:2])
    for x, y in zip(sim.inverse_read(), one.inverse_read()):
        assert np.array_equal(x[1:2].view(np.uint32), y.view(np.uint32))
    # transition Jacobians from a row that carries env 1's parameters, on a handle that has env 1's row in slot 0
    big = st.BatchedStepper(m, sim.fd_columns(False), lib_path=emu)
    ref = st.BatchedStepper(patched(m, p), sim.fd_columns(False), lib_path=emu)
    for name in st.PARAMS:
        big.param_set(name, p[name], env_ids=[0])
    for s in (big, ref):
        s.reset(q, v); s.set_control(np.full(m.nu, 0.1)); s.state_bank(1); s.save_state([0], [0])
        s.fd_transition([0], eps=1e-2, centered=False)
    for x, y in zip(big.fd_read(), ref.fd_read()):
        assert np.array_equal(x.view(np.uint32), y.view(np.uint32))
    with pytest.raises(st.StepperError, match='overlay'):
        sim.fd_inverse(q[None], v[None], qacc[:1], n=None)


def test_malformed_inputs_are_refused(emu):
    m = load_model('template')
    sim = st.BatchedStepper(m, 2, lib_path=emu)
    lib, h = sim._lib, sim._h
    k = lib.fb_param_size(h, 0)
    good = np.ones((2, k), np.float32)
    ids = np.array([0, 5], np.int32)
    assert lib.fb_param_size(h, 99) == -1 and lib.fb_param_size(h, -1) == -1
    cases = [(lambda: lib.fb_param_set(h, 12, None, 2, good.ctypes.data, 0), 'unknown parameter'),
             (lambda: lib.fb_param_set(h, 0, None, 1, good.ctypes.data, 0), 'n must be n_envs'),
             (lambda: lib.fb_param_set(h, 0, ids.ctypes.data, 2, good.ctypes.data, 0), 'env id out of range'),
             (lambda: lib.fb_param_set(h, 0, None, 2, None, 0), 'NULL')]
    for call, msg in cases:
        assert call() == -1 and msg in lib.fb_last_error(h).decode(), msg
    for name, bad, msg in (('body_mass', np.nan, 'non-finite'), ('dof_damping', -1.0, 'negative'), ('density', -1e-3, 'negative'),
                           ('geom_friction', np.inf, 'non-finite'), ('viscosity', -1.0, 'negative')):
        v = sim.param_get(name)
        v[0, 0] = bad
        with pytest.raises(st.StepperError, match=msg):
            sim.param_set(name, v)
    free = [j for j in range(m.njnt) if m.jnt_type[j] != 3][0]
    stiff = sim.param_get('jnt_stiffness'); stiff[:, free] = 1.0
    with pytest.raises(st.StepperError, match='not a hinge'):
        sim.param_set('jnt_stiffness', stiff)
    sim.param_set('gravity', [1.0, -2.0, 3.0])              # signed fields may be negative
    lo = nominal(m, 'body_mass')
    with pytest.raises(st.StepperError, match='lo > hi'):
        sim.param_draws('body_mass', lo, lo * 0.9)
    with pytest.raises(st.StepperError, match='negative'):
        sim.param_draws('body_mass', -lo - 1, lo)
    assert lib.fb_param_draws(h, 0, lo.astype(np.float32).ctypes.data, None, 0, 0) == -1
    with pytest.raises(KeyError):
        sim.param_set('body_pos', 0)
    env = fly_envs.template_task(n_envs=2, lib_path=emu)
    with pytest.raises(ValueError, match='shared'):
        env.randomize_model_params(shared=('body_mass',), dof_damping=(0, 1))
    env.close()


# ------------------------------------------------------------------------------------------------------------------------ GPU tier
@pytest.mark.gpu
@pytest.mark.parametrize('variant', ['template', 'flight'])
def test_overlay_steps_like_a_patched_model_on_gpu(variant):
    m = load_model(variant)
    n = 4096
    picks = [0, 1234, 4095]
    params = {k: random_params(m, 100 + k) for k in picks}
    sim = st.BatchedStepper(m, n)
    for k, p in params.items():
        for name in st.PARAMS:
            sim.param_set(name, p[name], env_ids=[k])
    q, v = start_state(m, 4)
    ctrl = np.random.RandomState(5).uniform(-0.5, 0.5, (n, m.nu))
    got = run(sim, q, v, ctrl, steps=4)
    ref = run(st.BatchedStepper(m, n), q, v, ctrl, steps=4)
    others = np.setdiff1d(np.arange(n), picks)
    for x, y in zip(got, ref):                              # the envs without parameters of their own: the null path's bits
        assert np.array_equal(x[others].view(np.uint32), y[others].view(np.uint32))
    for k, p in params.items():
        one = st.BatchedStepper(patched(m, p), 1)
        for x, y in zip(got, run(one, q, v, ctrl[k:k + 1], steps=4)):
            assert np.array_equal(x[k:k + 1].view(np.uint32), y.view(np.uint32)), (variant, k)
        one.close()
    mp = patched(m, params[1234])
    sim2 = st.BatchedStepper(m, 64)
    for name in st.PARAMS:
        sim2.param_set(name, params[1234][name], env_ids=[0])
    compare_stage_fields(mp, sim2, seed=3, env=0, act=True)


@pytest.mark.gpu
def test_draws_host_and_device_task_and_step_device_on_gpu():
    import torch
    n = 4096
    rs = np.random.RandomState(0)
    actions = rs.uniform(-0.5, 0.5, (22, n, 59)).astype(np.float32)
    rows = []
    for device_task in (False, True):
        env = fly_envs.template_task(n_envs=n, device_task=device_task, time_limit=0.02)
        m = env.model
        ranges = {k: (v[0] - 0.2 * np.abs(v[0]), v[0] + 0.2 * np.abs(v[0])) for k, v in env.model_params().items()}
        env.randomize_model_params(seed=9, shared=('body_mass', 'body_inertia'), **ranges)
        rows.append(drive_envs(env, actions))
        if device_task:
            stream = torch.cuda.ExternalStream(env._sim.stream)
            with torch.cuda.stream(stream):
                for k in range(12):
                    obs, out = env.step_device(torch.from_numpy(actions[k]).cuda())
                stream.synchronize()
            assert torch.isfinite(obs).all()
            for name, (lo, hi) in ranges.items():
                r = env.model_params()[name].reshape(n, -1)
                assert np.all(r >= np.float32(lo).reshape(-1)) and np.all(r <= np.float32(hi).reshape(-1)), name
            print('blocks per SM with the overlay:', {k: b for k, (_, b) in env._sim.step_kernel_smem().items()})
            assert min(b for _, b in env._sim.step_kernel_smem().values()) >= 8
        env.close()
    for a, b in zip(*rows):
        for name in st.PARAMS:
            assert np.array_equal(a[name], b[name]), name
