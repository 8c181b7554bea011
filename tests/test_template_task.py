"""template_task (reference fly_envs.py:249-300, tasks/template_task.py): the ghost-less walking model `fly_template.npz`, the contract of
the reference's installation test (tests/test_core.py), the model against the fp64 oracle, and the device task (kind 3) against the host
task code on the same stepper.  CPU tier: the host-emulation build.  GPU tier (-m gpu): rollouts, step_device, occupancy."""
import json
import os

import numpy as np
import pytest

import __graft_entry__ as ge
from flybody_b200 import fly_envs, stepper as st
from flybody_b200.dm_env_shim import StepType
from flybody_b200.flymodel import load_model, model_for, variant_name
from parity_common import compare_stage_fields, teacher_forced_errors, summarize_tf

OBS_NAMES = ['walker/' + s for s in ('accelerometer', 'actuator_activation', 'appendages_pos', 'force', 'gyro', 'joints_pos',
                                     'joints_vel', 'touch', 'velocimeter', 'world_zaxis')]      # reference tests/test_core.py:9-20
SHAPES = {'walker/actuator_activation': (59,), 'walker/appendages_pos': (21,), 'walker/force': (18,), 'walker/joints_pos': (85,), 'walker/joints_vel': (85,),
          'walker/touch': (6,)}


@pytest.fixture(scope='module')
def emu():
    ge.build()
    return ge.EMU


def test_template_model_is_the_walker_without_the_ghost():
    t, w = load_model('template'), load_model('walk')
    assert (t.nq, t.nv, t.nu) == (109, 108, 59)
    golden = json.load(open(os.path.join(os.path.dirname(__file__), 'golden', 'reference_goldens.json')))
    assert t.nv == golden['flybare_sizes']['nv']
    for key in ('body_names', 'jnt_names', 'site_names'):
        assert not [n for n in t.meta[key] if 'ghost' in n], key
    nb, nj, nq, nv, ns = t.nbody, t.njnt, t.nq, t.nv, t.nsite
    assert t.meta['body_names'] == w.meta['body_names'][:nb] and t.meta['jnt_names'] == w.meta['jnt_names'][:nj]
    walker = {'body': nb, 'jnt': nj, 'dof': nv, 'site': ns}
    # the compiler derives the invweights from the whole model's inertia at qpos0 and, for the filtered joints, stiffness and damping
    # from them: the ghost's absence moves those by rounding only
    derived = ('body_invweight0', 'dof_invweight0', 'jnt_stiffness', 'dof_damping')
    for k, v in t.a.items():
        if not isinstance(v, np.ndarray) or k not in w.a or k == 'body_subtreemass':
            continue
        pre = k.split('_')[0]
        n = nq if k in ('qpos0', 'qpos_spring') else walker.get(pre)
        ref = w.a[k][:n] if n is not None and v.shape[0] == n else w.a[k]
        assert v.shape == ref.shape, k
        if k in derived:
            assert np.allclose(v, ref, rtol=1e-8, atol=0), k
        else:
            assert np.array_equal(v, ref), k
    assert np.array_equal(t.body_subtreemass[1:], w.body_subtreemass[1:nb])        # the world's subtree lost the ghost only
    assert model_for('template').nv == 108
    assert variant_name('template') == 'fly_template' and variant_name('walk', joint_filter=0.02) == 'fly_walk_jf0.02'
    assert variant_name('template', adhesion_filter=0.01) == 'fly_template_af0.01'


def test_template_model_equals_a_compile_without_the_ghost():
    """the model cut from the walk model against the project's compiler run on the reference's fruitfly.xml with add_ghost=False
    (compile_variant('template')), where that file is reachable"""
    from oracle.variants import assets_dir
    src = assets_dir()
    if src is None:
        pytest.skip("the reference's fruitfly.xml is not reachable (FLYBODY_ASSETS, an installed flybody, FLYBODY_REFERENCE)")
    from flybody_b200.compiler import compile_model as cm
    from flybody_b200.flymodel import from_compiled
    c, t = from_compiled(cm.compile_variant('template', assets_dir=src, mesh_cache=cm.load_mesh_cache(src))), load_model('template')
    skip = ('ngeom_all', 'stat_meaninertia')             # (ngeom_all counts visual geoms: not part of the cut model)
    assert {k: v for k, v in c.meta.items() if k not in skip} == {k: v for k, v in t.meta.items() if k not in skip}
    assert abs(t.meta['stat_meaninertia'] - c.meta['stat_meaninertia']) <= 1e-12 * c.meta['stat_meaninertia']
    assert set(c.a) == set(t.a) | {'ngeom_all'}
    for k, v in c.a.items():
        if isinstance(v, np.ndarray):                       # invweight-derived arrays: the ghost's tree moves them by rounding only
            assert v.shape == t.a[k].shape and np.allclose(v, t.a[k], rtol=1e-12, atol=0), k


@pytest.mark.parametrize('n_envs', [None, 3])
def test_core_contract(emu, n_envs):
    """reference tests/test_core.py::test_can_create_and_run_environment, batched and single"""
    env = fly_envs.template_task(n_envs=n_envs, lib_path=emu)
    assert list(env.observation_spec()) == OBS_NAMES
    assert env.action_spec().shape == (59,)
    ts = env.reset()
    lead = () if n_envs is None else (n_envs,)
    for name in OBS_NAMES:
        assert isinstance(ts.observation[name], (float, np.ndarray))
        assert ts.observation[name].shape == lead + SHAPES.get(name, (3,)), name
    rs = np.random.RandomState(0)
    for _ in range(100):
        ts = env.step(rs.uniform(-1, 1, lead + (59,)))
        assert np.all(np.asarray(ts.reward) == 1)
    env.close()


def test_action_corruptor(emu):
    """reference tests/test_core.py::test_action_corruptor against env.prev_action"""
    env = fly_envs.template_task(lib_path=emu)
    env.reset()
    rs = np.random.RandomState(1)
    for _ in range(20):
        a = rs.uniform(-1, 1, 59)
        env.step(a)
        assert np.allclose(a, env.prev_action)
    noise = rs.normal(scale=0.1, size=59)
    seen = []
    env = fly_envs.template_task(lib_path=emu, action_corruptor=lambda a, r: (seen.append(r), a + noise)[1])
    env.reset()
    for _ in range(20):
        a = rs.uniform(-1, 1, 59)
        env.step(a)
        assert np.allclose(a + noise, env.prev_action)
    assert isinstance(seen[0], np.random.RandomState)
    env.close()


def test_unsupported_options_raise(emu):
    with pytest.raises(NotImplementedError, match='set_applied_forces'):
        fly_envs.template_task(mjcb_control=lambda m, d: None, lib_path=emu)
    with pytest.raises(NotImplementedError):
        fly_envs.template_task(observables_options={'joints_pos': {'enabled': False}}, lib_path=emu)
    env = fly_envs.template_task(n_envs=2, lib_path=emu, device_task=True, action_corruptor=lambda a, r: a)
    with pytest.raises(RuntimeError):
        env.step_device(np.zeros((2, 59), np.float32))
    env.close()


def test_template_model_matches_oracle(emu):
    m = load_model('template')
    for seed in (0, 1):
        compare_stage_fields(m, st.BatchedStepper(m, 2, lib_path=emu), seed=seed, act=True)
    r = summarize_tf(*teacher_forced_errors(m, st.BatchedStepper(m, 1, lib_path=emu), n_steps=8, n_sub=10))
    assert r['p90_q'] < 2e-6 and r['p90_v'] < 2e-3 and r['hist_v']['<0.005'] >= 7, r      # the walk gates (test_emu_parity.py)
    assert r['p90_s'] < 1e-3, r


def test_env_applied_forces_are_zeroed_by_resets(emu):
    env = fly_envs.template_task(n_envs=3, lib_path=emu, time_limit=0.01)      # 5 control steps
    env.reset()
    m = env.model
    env.set_applied_forces(qfrc=np.full(m.nv, 1e-5), xfrc=np.full((m.nbody, 6), 1e-5), env_ids=[0, 2])
    q, x = env._sim.applied()
    assert q[0].all() and not q[1].any() and x[2].all()
    for _ in range(5):
        ts = env.step(np.zeros((3, 59)))
    assert np.all(np.asarray(ts.step_type) == int(StepType.LAST)) and np.all(ts.discount == 1)
    q, _ = env._sim.applied()
    assert q[0].all()                                       # persist through the episode ...
    ts = env.step(np.zeros((3, 59)))
    q, x = env._sim.applied()
    assert np.all(np.asarray(ts.step_type) == int(StepType.FIRST)) and not q.any() and not x.any()      # ... zeroed by the auto-reset
    env.set_applied_forces(qfrc=np.ones(m.nv))
    env.clear_applied_forces()
    assert not env._sim.applied()[0].any()
    env.close()


def drive(env, actions):
    """step a device-task template env and re-derive, from the same observation record, what the host task code gives"""
    ts = env.reset()
    assert np.all(np.asarray(ts.step_type) == int(StepType.FIRST))
    seen = [np.asarray(ts.step_type, np.int64)]
    time = np.zeros(env.n_envs)
    for k in range(len(actions)):
        resetting = env._needs_reset.copy()
        ts = env.step(actions[k])
        time = np.where(resetting, 0.0, time + env._control_timestep)
        obs = env._observation(env._rec)
        step_type, reward, discount, needs = env._task_after(env._rec, obs, resetting, time, None)
        assert np.array_equal(np.asarray(step_type, np.int64), np.asarray(ts.step_type, np.int64)), (k, step_type, ts.step_type)
        assert np.array_equal(reward, ts.reward) and np.array_equal(discount, ts.discount), k
        assert np.array_equal(needs, env._needs_reset), k
        if resetting.any():                                 # the template pose at rest
            q, v = env._sim.get(st.QPOS)[resetting], env._sim.get(st.QVEL)[resetting]
            assert np.allclose(q, env.model.qpos0.astype(np.float32)) and not v.any(), k
        seen.append(np.asarray(ts.step_type, np.int64))
    return np.array(seen)


def test_device_task_matches_host_task_code(emu):
    n = 4
    rs = np.random.RandomState(0)
    actions = rs.uniform(-0.5, 0.5, (30, n, 59)).astype(np.float32)
    actions[:, 2] = 1e12                                    # env 2 thrashes: |qacc| > _TERMINAL_QACC, discount 0
    actions[4, 1, 7] = np.nan
    env = fly_envs.template_task(n_envs=n, lib_path=emu, device_task=True, time_limit=0.02)      # LAST at step 10
    env.set_applied_forces(xfrc=np.ones((env.model.nbody, 6)) * 1e-3)
    seen = drive(env, actions)
    assert (seen[:, 2] == int(StepType.LAST)).any() and (seen[:, 2] == int(StepType.FIRST)).sum() > 2
    assert np.all(seen[[10, 21], 0] == int(StepType.LAST)) and np.all(seen[[11, 22], 0] == int(StepType.FIRST))
    assert not env._sim.applied()[1].any()                  # the device resets zeroed the applied forces
    env.close()


# ------------------------------------------------------------------------------------------------------------------------ GPU tier
@pytest.mark.gpu
def test_random_rollout_4096_envs_on_gpu():
    env = fly_envs.template_task(n_envs=4096, device_task=True, seed=1)
    env.reset()
    rs = np.random.RandomState(0)
    for _ in range(20):
        ts = env.step(rs.uniform(-1, 1, (4096, 59)).astype(np.float32))
    q, v = env._sim.get(st.QPOS), env._sim.get(st.QVEL)
    assert np.all(np.isfinite(q)) and np.all(np.isfinite(v))
    rq = env._root_q
    assert np.abs(np.linalg.norm(q[:, rq + 3:rq + 7], axis=1) - 1).max() < 1e-5
    assert np.all(np.asarray(ts.reward)[np.asarray(ts.step_type) != int(StepType.FIRST)] == 1)
    env.close()


@pytest.mark.gpu
def test_step_device_matches_step_on_gpu():
    import torch
    n = 64
    a_env = fly_envs.template_task(n_envs=n, device_task=True, time_limit=0.02)
    b_env = fly_envs.template_task(n_envs=n, device_task=True, time_limit=0.02)
    a_env.reset(); b_env.reset()
    stream = torch.cuda.ExternalStream(a_env._sim.stream)
    lay = a_env.observation_layout()
    assert list(lay) == OBS_NAMES
    rs = np.random.RandomState(0)
    for k in range(25):
        act = rs.uniform(-1, 1, (n, 59)).astype(np.float32)
        ts = b_env.step(act)
        with torch.cuda.stream(stream):
            obs, out = a_env.step_device(torch.from_numpy(act).cuda())
            stream.synchronize()
            obs_h, out_h = obs.cpu().numpy(), out.cpu().numpy()
        assert np.array_equal(out_h[:, 2].astype(np.int64), np.asarray(ts.step_type, np.int64)), k
        assert np.array_equal(out_h[:, 0], np.asarray(ts.reward, np.float32)) and np.array_equal(out_h[:, 1], np.asarray(ts.discount, np.float32))
        for key in OBS_NAMES:
            sl, shp = lay[key]
            assert np.array_equal(obs_h[:, sl].reshape((n,) + shp), ts.observation[key]), (k, key)
    a_env.close(); b_env.close()


@pytest.mark.gpu
def test_step_kernels_reach_the_compiled_blocks_per_sm_on_gpu():
    import torch
    from test_model_variants import compiled_min_blocks, SM90_SMEM_PER_CTA_RESERVED, STEP_KERNELS
    props = torch.cuda.get_device_properties(0)
    minb = compiled_min_blocks()
    sim = st.BatchedStepper(load_model('template'), 4096)
    budget = sim.step_kernel_smem()
    sim.close()
    print('blocks per SM template:', {k: v[1] for k, v in budget.items()})
    assert set(budget) == STEP_KERNELS
    for kname, (nbytes, blocks) in budget.items():
        assert (nbytes + SM90_SMEM_PER_CTA_RESERVED) * minb <= props.shared_memory_per_multiprocessor, (kname, nbytes, props.name)
        assert blocks >= minb, (kname, nbytes, blocks, props.name)
