"""State rows (fb_state_*; env.state_bank / save_state / load_state / state_dict): an env taken out of the stepper and put back -- into
the same env, another env, or a fresh stepper -- continues bit for bit.  "Equal" is array_equal on raw bits (uint32 views, so NaNs
count), never a tolerance.  CPU tier: the host-emulation build of the kernel source; GPU tier (-m gpu): the same checks on the device."""
import numpy as np
import pytest

import __graft_entry__ as ge
from flybody_b200 import fly_envs, stepper as st
from flybody_b200.flymodel import load_model

GETS = (st.QPOS, st.QVEL, st.ACT, st.CTRL, st.QACC, st.TIME, st.FLAGS, st.SENSORDATA, st.SENSOR_MEAN, st.NCON, st.NEFC, st.XPOS,
        st.SITE_XPOS, st.SUBTREE_COM, st.QFRC_BIAS, st.QFRC_PASSIVE, st.CONTACT)


@pytest.fixture(scope='module')
def emu():
    ge.build()
    return ge.EMU


@pytest.fixture(scope='module')
def datasets(emu, tmp_path_factory):
    """the synthetic flight and walking datasets of the dataset tests"""
    from test_device_dataset_flight import write_dataset
    from test_device_dataset_walk import record_dataset
    d = tmp_path_factory.mktemp('state_datasets')
    paths = {'flight': str(d / 'flight.npz'), 'walk': str(d / 'walk.npz')}
    write_dataset(paths['flight'])
    record_dataset(emu, paths['walk'])
    return paths


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a.view(np.uint64) if a.dtype == np.float64 else a


def same(a, b, what=''):
    a, b = bits(np.asarray(a)), bits(np.asarray(b))
    assert a.shape == b.shape and np.array_equal(a, b), (what, np.argwhere(a != b)[:5])


def make(kind, lib, n, datasets=None, **kw):
    kw = dict(n_envs=n, lib_path=lib, seed=5, device_task=True) | kw
    if kind == 'walk':
        return fly_envs.walk_imitation(terminal_com_dist=0.3, **kw)
    if kind == 'walk_host':
        return fly_envs.walk_imitation(reset_noise=0.02, **(kw | dict(device_task=False)))
    if kind == 'flight':
        return fly_envs.flight_imitation(**kw)
    if kind == 'template':
        return fly_envs.template_task(time_limit=0.05, **kw)
    if kind == 'ball':
        return fly_envs.walk_on_ball(**kw)
    if kind == 'vision':
        return fly_envs.vision_guided_flight(terrain_bank=3, **kw)
    if kind == 'flight_dataset':
        return fly_envs.flight_imitation(ref_path=datasets['flight'], traj_indices=[0, 1, 3, 1], randomize_start_step=True, terminal_com_dist=0.02, **kw)
    if kind == 'walk_dataset':
        return fly_envs.walk_imitation(ref_path=datasets['walk'], traj_indices=[0, 1, 3, 1, 4], terminal_com_dist=0.05, **kw)
    raise KeyError(kind)


def actions(env, n_steps, seed=0, amp=0.3):
    rs = np.random.RandomState(seed)
    a = rs.uniform(-amp, amp, (n_steps, env.n_envs, env.action_spec().shape[0])).astype(np.float32)
    a[min(3, n_steps - 1), 0, 0] = np.nan                          # a NaN action acts as 0, on both sides
    return a


def snap(env, scratch):
    """everything observable of the env batch: the state rows of all envs (saved into scratch slots: integrated state, warm start, sensor
    sums, observation rows, `out`, task state) and the recomputed fields fb_get serves"""
    sim = env._sim
    ids = np.arange(env.n_envs)
    sim.save_state(scratch + ids, ids)
    out = {'rows': sim.read_states(scratch + ids)}
    for f in GETS:
        out[f] = sim.get(f).copy()
    return out


def same_snap(a, b, envs=None, what=''):
    for k in a:
        same(a[k] if envs is None else a[k][envs], b[k] if envs is None else b[k][envs], (what, k))


def same_ts(a, b, what=''):
    same(np.asarray(a.step_type), np.asarray(b.step_type), (what, 'step_type'))
    same(np.asarray(a.reward, np.float64), np.asarray(b.reward, np.float64), (what, 'reward'))
    same(np.asarray(a.discount, np.float64), np.asarray(b.discount, np.float64), (what, 'discount'))
    for k in a.observation:
        same(a.observation[k], b.observation[k], (what, k))


def roll(env, acts, every=None):
    out = []
    for t, a in enumerate(acts):
        ts = env.step(a)
        ts = ts._replace(observation={k: np.array(v) for k, v in ts.observation.items()})      # (the env's rows are views of one buffer)
        out.append(ts)
        if every is not None:
            every(t, ts)
    return out


def prepared(kind, lib, n, datasets, pre, seed=1):
    """an env mid-episode after `pre` control steps of random actions, one env freshly reset and one waiting for its reset, with a bank of 2 n slots"""
    env = make(kind, lib, n, datasets)
    env.reset()
    roll(env, actions(env, pre, seed))
    env.request_reset([n - 1])
    env.step(actions(env, 1, seed + 50)[0])
    env.request_reset([1])
    env.state_bank(2 * n)
    return env


def run_round_trip(kind, lib, n, datasets, pre, post):
    env, twin = prepared(kind, lib, n, datasets, pre), prepared(kind, lib, n, datasets, pre)
    before = snap(env, n)
    stale = {f: env._sim.get(f).copy() for f in (st.QFRC_SMOOTH, st.QFRC_CONSTRAINT, st.EFC_FORCE)}
    env.save_state()
    env.load_state(np.arange(n), np.arange(n))
    same_snap(before, snap(env, n), what='after load')
    for f, v in stale.items():
        same(v, env._sim.get(f), f)
    acts = actions(env, post, 9)
    for t, (a, b) in enumerate(zip(roll(env, acts), roll(twin, acts))):
        same_ts(a, b, t)
    same_snap(snap(env, n), snap(twin, n), what='end')
    env.close(); twin.close()


def test_round_trip_is_exact(emu):
    run_round_trip('walk', emu, 3, None, 30, 20)


def run_fresh(kind, lib, n, datasets, pre, post, tmp_path):
    """handle A rolled out, its state_dict through np.savez into a new env object that never stepped: both agree on every later step"""
    a = prepared(kind, lib, n, datasets, pre)
    np.savez(str(tmp_path / 'state.npz'), **a.state_dict())
    with np.load(str(tmp_path / 'state.npz')) as z:
        d = {k: z[k] for k in z.files}
    b = make(kind, lib, n, datasets)
    b.state_bank(2 * n)
    b.load_state_dict(d)
    same_snap(snap(a, n), snap(b, n), what='loaded')
    acts = actions(a, post, 11)
    firsts = 0
    for t, x in enumerate(acts):
        if t == post // 2:
            a.request_reset([0]); b.request_reset([0])
        ta, tb = a.step(x), b.step(x)
        same_ts(ta, tb, t)
        firsts += int((np.asarray(ta.step_type) == 0).sum())
        if t % 10 == 0 or t == post - 1:
            same_snap(snap(a, n), snap(b, n), what=t)
    assert firsts >= 2                                            # the env waiting for its reset, and at least one reset later
    a.close(); b.close()


@pytest.mark.parametrize('kind', ['walk', 'flight', 'template', 'ball', 'vision', 'flight_dataset', 'walk_dataset', 'walk_host'])
def test_fresh_env_continues(emu, datasets, tmp_path, kind):
    run_fresh(kind, emu, 3, datasets, 30, 50, tmp_path)


def test_rewind(emu):
    n, k = 3, 12
    env = prepared('flight', emu, n, None, 30)
    env.save_state()
    rng = env._rs.get_state()                                     # the wing-beat phase of a reset is drawn on the host: not part of a slot
    acts = actions(env, k, 4)
    first = roll(env, acts)
    end = snap(env, n)
    env.load_state(np.arange(n), np.arange(n))
    env._rs.set_state(rng)
    for t, (a, b) in enumerate(zip(first, roll(env, acts))):
        same_ts(a, b, t)
    same_snap(end, snap(env, n))
    env.close()


def run_fan_out(lib, n, targets, source, pre, post):
    env, twin = prepared('template', lib, n, None, pre), prepared('template', lib, n, None, pre)
    targets = np.asarray(targets)
    others = np.setdiff1d(np.arange(n), targets)
    env.save_state(slots=[0], env_ids=[source])
    env.load_state(np.zeros(len(targets), np.int64), targets)
    same_snap(snap(env, n), snap(twin, n), envs=others, what='isolation at the load')
    acts = actions(env, post, 6)
    acts[:, targets] = acts[:, [source]]                          # equal actions for the copies and their source
    for t in range(post):
        ta, tb = env.step(acts[t]), twin.step(acts[t])
        for k in ta.observation:
            same(ta.observation[k][others], tb.observation[k][others], ('isolation', t, k))
            same(ta.observation[k][targets], np.broadcast_to(tb.observation[k][source], ta.observation[k][targets].shape), ('fan-out', t, k))
        same(np.asarray(ta.step_type)[targets], np.full(len(targets), np.asarray(tb.step_type)[source]), t)
    a, b = snap(env, n), snap(twin, n)
    same_snap(a, b, envs=others, what='isolation at the end')
    for f in (st.QPOS, st.QVEL, st.QACC, st.NCON, st.NEFC):
        same(a[f][targets], np.broadcast_to(b[f][source], a[f][targets].shape), f)
    env.close(); twin.close()


def test_fan_out_and_isolation(emu):
    run_fan_out(emu, 8, [1, 5, 6, 7], 2, 20, 10)


def test_applied_forces_travel_with_the_row(emu):
    n = 3
    m = load_model('template')
    env = make('template', emu, n)
    env.reset()
    sig0, slots0 = env._sim.state_signature(), env._sim.state_slots
    x = np.zeros((n, m.nbody, 6), np.float32)
    x[1, m.body_id('walker/thorax'), 2] = 3.0
    env.set_applied_forces(qfrc=np.full(m.nv, 0.01, np.float32), xfrc=x)
    assert env._sim.state_signature() != sig0 and env._sim.state_slots > slots0      # the rows carry them only when the handle has them
    roll(env, actions(env, 5, 1))
    env.state_bank(n)
    env.save_state()
    saved = [v.copy() for v in env._sim.applied()]
    env.set_applied_forces(qfrc=np.zeros(m.nv, np.float32), xfrc=np.zeros_like(x))
    acts = actions(env, 5, 2)
    unforced = roll(env, acts)
    env.load_state(np.arange(n), np.arange(n))
    for a, b in zip(saved, env._sim.applied()):
        same(a, b, 'applied forces after the load')
    forced = roll(env, acts)
    assert not np.array_equal(forced[-1].observation['walker/joints_pos'], unforced[-1].observation['walker/joints_pos'])
    env.clear_applied_forces()                                    # back on the path without the term: the layout changed, the bank is gone
    assert env._sim.state_signature() == sig0
    with pytest.raises(st.StepperError, match='dropped'):
        env.save_state()
    env.close()


def test_errors(emu):
    n = 3
    env = make('template', emu, n)
    with pytest.raises(RuntimeError, match='state_bank'):
        env.save_state()
    env.reset()
    sim = env._sim
    with pytest.raises(st.StepperError, match='no state bank'):
        sim.save_state()
    env.state_bank(4)
    for bad in (dict(slots=[4], env_ids=[0]), dict(slots=[-1], env_ids=[0]), dict(slots=[0], env_ids=[n]), dict(slots=[1, 1], env_ids=[0, 1])):
        with pytest.raises(st.StepperError):
            sim.save_state(**bad)
    sim.save_state(slots=[0], env_ids=[1])
    with pytest.raises(st.StepperError, match='never written'):
        sim.load_state([1], [0])
    with pytest.raises(st.StepperError, match='never written'):
        sim.read_states([2])
    with pytest.raises(st.StepperError, match='twice'):
        sim.load_state([0, 0], [2, 2])
    with pytest.raises(st.StepperError, match='out of range'):
        sim.load_state([0], [n])
    with pytest.raises(ValueError):
        sim.write_states([0], np.zeros((1, 3), np.uint32))
    with pytest.raises(st.StepperError, match='does not fit|out of memory'):
        sim.state_bank(2 ** 31 - 1)
    env.state_bank(4)
    env.save_state(slots=[0], env_ids=[1])
    env._program_ref_id = None
    env._upload_program()                                         # the programs are replaced: the bank is stale
    with pytest.raises(st.StepperError, match='dropped'):
        env.load_state([0], [0])
    env.state_bank(n)
    other = make('walk', emu, n)
    with pytest.raises(ValueError, match='signature'):
        other.load_state_dict(env.state_dict())
    env.close(); other.close()


def test_host_side_dataset_and_vision_are_refused(emu, datasets):
    env = fly_envs.flight_imitation(ref_path=datasets['flight'], traj_indices=[0, 1], n_envs=2, lib_path=emu)
    with pytest.raises(NotImplementedError, match='device_task=True'):
        env.state_bank(2)
    env.close()
    env = fly_envs.vision_guided_flight(n_envs=2, lib_path=emu)
    with pytest.raises(NotImplementedError, match='device_task=True'):
        env.state_dict()
    env.close()


def test_save_and_load_leave_the_step_launches_alone(emu):
    n = 3
    env = prepared('walk', emu, n, None, 3)
    sim = env._sim
    a = actions(env, 4, 3)
    c0 = sim.launch_count; env.step(a[0]); per_step = sim.launch_count - c0
    c0 = sim.launch_count; env.save_state(); assert sim.launch_count - c0 == 1
    c0 = sim.launch_count; env.step(a[1]); assert sim.launch_count - c0 == per_step
    c0 = sim.launch_count; env.load_state([0], [2]); assert sim.launch_count - c0 == 1 + 4      # the copy, then pos, col, proj, vel of one env
    c0 = sim.launch_count; env.step(a[2]); assert sim.launch_count - c0 == per_step
    env.close()


# ---------------------------------------------------------------------------------------------------------------- GPU tier
@pytest.mark.gpu
def test_gpu_round_trip_is_exact():
    run_round_trip('walk', None, 4096, None, 30, 20)


@pytest.mark.gpu
@pytest.mark.parametrize('kind', ['walk', 'flight', 'template', 'ball', 'vision', 'flight_dataset', 'walk_dataset', 'walk_host'])
def test_gpu_fresh_env_continues(emu, datasets, tmp_path, kind):
    run_fresh(kind, None, 64, datasets, 30, 50, tmp_path)


@pytest.mark.gpu
def test_gpu_fan_out_and_isolation():
    n = 4096
    targets = np.unique(np.concatenate([[1, 5, 6, 4095], np.random.RandomState(0).choice(n, n // 20, replace=False)]))
    run_fan_out(None, n, targets[targets != 2], 2, 20, 10)


@pytest.mark.gpu
def test_gpu_step_launches_survive_save_and_load():
    """a control step between saves and loads (one env list, all envs) launches what it launched before"""
    n = 256
    env = prepared('walk', None, n, None, 6)
    sim = env._sim
    a = actions(env, 6, 3)
    env.step(a[0])
    sim.sync()
    c0 = sim.launch_count; env.step(a[1]); per_step = sim.launch_count - c0
    env.save_state()
    env.load_state(np.arange(8), np.arange(8) + 100)
    env.load_state(np.arange(n), np.arange(n))
    for k in range(2, 5):
        c0 = sim.launch_count; env.step(a[k]); assert sim.launch_count - c0 == per_step
    env.close()
