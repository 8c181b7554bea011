"""The smooth half of the step against the fp64 oracle, element by element (tests/smooth_states.py): kinematics, composite inertia, the
L^T D L factorisations of M and of M + hD with their triangular sweeps, RNE bias, springs, dampers, inertia-box and ellipsoid fluid,
actuation and sensors, on the constraint-free copies of walk, flight, vision, the ball model and the FruitFly variants, at pinned
states that reach the edges: uniformly random root quaternions (one a 180-degree turn, -q, 0.5 q and 2 q), hinges across their whole
range, the root 1e2 and 1e3 cm from the origin, wings at real wing-beat speeds, the body at the flight task's termination speeds, and
nonzero activations.

Gates (fp32 stepper vs fp64 oracle; tolerance = measured x 2.5, the measurement is printed, one row per state):
  qM                               max_ij |dM_ij| / sqrt(M_ii M_jj)                                                  QM
  bias, passive, actuator, smooth  max_i |df_i| / sqrt(M_ii), relative to max_j |f_j| / sqrt(M_jj)                 FORCE
  qacc (nefc = 0)                  backward: max_i |(M qacc_dev - qfrc_smooth)_i| / (|M| |qacc_dev| + |qfrc_smooth|)_i  BACK
                                   forward: max_i |dqacc_i| sqrt(M_ii), relative to max_j |qacc_j| sqrt(M_jj)        FWD
  one substep's dqvel / h          the same two, for M + h diag(damping)                                            BACK, FWD
  both solves, probe right-hand    qfrc_applied chosen so that every dof's solution is 1 in the inertia metric; per  PROBE
  side                             dof |dx_i| sqrt(A_ii) against the fp64 solve of the stepper's own M (and M + hD)
  xpos, site_xpos, subtree_com     |dx| / (distance from the root + 1e-2 cm) where |x| < 10 cm                     POS
                                   |dx| in units of 2^-24 max(|x|, 1 cm), everywhere (the far states)               POS_ULPS
  xmat, site_xmat                  max |dR_ij|                                                                      XMAT
  sensordata                       per sensor |ds| / (max |s| + parity_common.SENSOR_FLOOR[type])                  SENSOR
  fluid                            qfrc_passive with the medium on minus off, per dof in the inertia metric        FLUID
"""
import numpy as np
import pytest

import __graft_entry__ as ge
import smooth_states as ss
from flybody_b200 import stepper as st

# measured under emulation (the kernel source on the host) and on an H100 (80 GB HBM3, 700 W power limit), the larger of the two x 2.5;
# the worst state / model of the larger in parentheses
TOL = dict(
    qM=2e-6,                 # H100 7.8e-7 (ball wings_only), emulation 6.3e-7
    qfrc_bias=3.4e-6,        # H100 1.32e-6, emulation 1.36e-6 (walk_wings flight)
    qfrc_passive=4.3e-6,     # H100 1.69e-6 (walk flight), emulation 1.62e-6
    qfrc_actuator=1.9e-7,    # H100 and emulation 7.7e-8 (ball quat_w0)
    qfrc_smooth=3.4e-6,      # H100 and emulation 1.34e-6 (walk_force flight)
    xpos=5e-6, site_xpos=5e-6, subtree_com=5e-6,                 # H100 1.8e-6, emulation 2.0e-6 (ball quat_b)
    xpos_ulps=3.2, site_xpos_ulps=3.2, subtree_com_ulps=3.2,      # H100 1.14, emulation 1.25 (walk flight)
    xmat=1.2e-6,             # H100 4.0e-7, emulation 4.7e-7 (walk wings_only)
    sensor=2.6e-5,           # H100 1.02e-5 (walk flight), emulation 8.9e-6
    qacc_back=6.3e-6,        # H100 2.52e-6 (walk_jf0 flight), emulation 2.36e-6
    qacc_fwd=3.1e-6,         # H100 and emulation 1.22e-6 (walk_force flight)
    dv_back=1.2e-5,          # H100 4.66e-6 (walk_jf0 body_only), emulation 4.50e-6
    dv_fwd=3.2e-6,           # H100 and emulation 1.26e-6 (walk flight)
    fluid=2.1e-6,            # flight models (ellipsoid wings, inertia-box body): emulation 8.2e-7 (flight_legs body_only), H100 4.2e-7
    # walking models (inertia-box drag on every body, the wings included): 3.07e-5 on the H100 and under emulation at wing-beat speeds
    # (walk wings_only), 5.6e-6 at the termination speeds (body_only).  The cause: body_fluid_wrench (fb_tree.h) rebuilds the box sides
    # sqrt(6 (I_j + I_k - I_i) / m) from the fp32 body_inertia, and a wing is a thin plate whose thin side cancels (1.7e-3 relative,
    # every other body <= 3e-6).  Box sides computed in fp64 on the host bring this to 8.3e-7, but move two chaotic teacher-forced
    # checks (test_walk_on_ball.py ball_wings, test_gpu_parity.py walk) across their contact-event thresholds: not changed here
    fluid_box=7.8e-5,
    # solves on a right-hand side that gives every dof a solution of size 1 in the inertia metric, against the fp64 solve of the
    # stepper's own M (smooth_states.probe_solve_errors): the factorisation and its sweeps alone.  Emulation 1.44e-6 (walk_wings) /
    # 1.20e-6 (flight_legs); a factorisation-schedule item dropped at the first step gives 5.3e-6 - 1.0e-5 there.  The H100 (FMA
    # contraction) measures up to 2.75e-6 / 1.67e-6: its own tolerances below
    probe_qacc=3.6e-6,
    probe_dv=3.0e-6,
)
TOL_H100 = dict(TOL, probe_qacc=6.9e-6, probe_dv=4.2e-6)
PRE_CONSTRAINT = ('qM', 'qfrc_bias', 'qfrc_passive', 'qfrc_actuator', 'qfrc_smooth', 'xpos', 'site_xpos', 'subtree_com',
                  'xpos_ulps', 'site_xpos_ulps', 'subtree_com_ulps', 'xmat')
GPU_MODELS = ss.MODELS

_ORACLE = {}


def model(name, free=True, fluid=True, springs=True):
    m = ss.base_model(name)
    return ss.free_model(m, fluid=fluid, springs=springs) if free else m


def oracle(name, free=True, fluid=True, springs=True):
    """oracle fields of every applicable state of model `name` (cached: the oracle is deterministic)"""
    key = (name, free, fluid, springs)
    if key not in _ORACLE:
        m = model(name, free, fluid, springs)
        _ORACLE[key] = {k: ss.oracle_fields(m, k, step=springs) for k in ss.state_names(m)}
    return _ORACLE[key]


def gate(label, name, sim, m, assign=None, keys=None, free=True):
    """run the states of model `name` on `sim` (env i holds state names[assign[i]]; default one env per state), gate every env and
    print one row per state (its worst env)"""
    names = ss.state_names(m)
    assign = list(range(len(names))) if assign is None else assign
    ora = oracle(name, free)
    dev = ss.device_fields(m, sim, names, assign)
    keys = keys or [k for k in TOL if not k.startswith('fluid')]
    probe = ss.probe_solve_errors(m, sim, names, assign) if free else None
    worst, bad = {}, []
    for i, d in enumerate(dev):
        k = names[assign[i]]
        o = ora[k]
        assert d['flags'] == 0, (label, k, i, d['flags'])
        if free:
            assert d['nefc'] == o['nefc'] == 0, (label, k, i, d['nefc'], o['nefc'])
        e = ss.errors(m, d, o)
        if probe:
            e['probe_qacc'], e['probe_dv'] = probe[i]
        w = worst.setdefault(k, {})
        for key in keys:
            if key in e:
                w[key] = max(w.get(key, 0.0), e[key])
                if not e[key] < (TOL_H100 if label.startswith('H100') else TOL)[key]:
                    bad.append((k, i, key, e[key]))
    print(f'\n{label}: {len(dev)} envs')
    cols = [c for c in keys if any(c in w for w in worst.values())]
    print('  ' + f'{"state":<12}' + ''.join(f'{c[:11]:>12}' for c in cols))
    for k, w in worst.items():
        print('  ' + f'{k:<12}' + ''.join(f'{w.get(c, float("nan")):12.2e}' for c in cols))
    assert not bad, (label, bad[:8])
    return worst


def fluid_models(name):
    """(medium on, medium off), both without joint springs and dampers"""
    return model(name, springs=False), model(name, fluid=False, springs=False)


def fluid_gate(label, name, sims):
    """the fluid part of qfrc_passive (medium on minus off, the same model edits on both sides) on the states where only the wings or
    only the body move, per dof in the inertia metric; sims: steppers on fluid_models(name)"""
    m_on, m_off = fluid_models(name)
    names = [k for k in ss.FLUID_STATES if ss.applies(m_on, k)]
    on, off = oracle(name, springs=False), oracle(name, fluid=False, springs=False)
    every = ss.state_names(m_on)
    d_on = ss.device_fields(m_on, sims[0], every, list(range(len(every))), step=False)
    d_off = ss.device_fields(m_off, sims[1], every, list(range(len(every))), step=False)
    out = {}
    print(f'\n{label}')
    for k in names:
        a, b = d_on[every.index(k)], d_off[every.index(k)]
        assert not b['qfrc_passive'].any() and not off[k]['qfrc_passive'].any(), (label, k)
        fo_ = on[k]['qfrc_passive'] - off[k]['qfrc_passive']
        fd = a['qfrc_passive'] - b['qfrc_passive']
        M = on[k]['qM'].reshape(m_on.nv, m_on.nv)
        out[k] = e = ss.force_error(fd, fo_, M)
        key = 'fluid_box' if m_on.nfluid == 0 else 'fluid'
        print(f'  {k:<12} max |fluid force| {np.abs(fo_).max():9.2e}, error {e:9.2e} ({key})')
        assert np.abs(fo_).max() > 0, (label, k)
        assert e < TOL[key], (label, k, e)
    return out


def gate_twins(label, m, sim):
    """-q, 0.5 q and 2 q give the fields of q, and the far states those of the state at the origin, within the gates (stepper vs
    stepper: the kinematics normalise the quaternion, and the kernels work relative to the root)"""
    names = ss.state_names(m)
    dev = dict(zip(names, ss.device_fields(m, sim, names, list(range(len(names))))))
    twins = [k for k in ('quat_neg', 'quat_half', 'quat_double', 'far_1e2', 'far_1e3') if k in dev]
    print(f'\n{label}: against quat_a')
    for k in twins:
        e = ss.errors(m, dev[k], dev['quat_a'])
        keys = [c for c in ('qM', 'qfrc_bias', 'qfrc_passive', 'qfrc_actuator', 'qfrc_smooth', 'qacc_fwd', 'dv_fwd', 'xmat', 'sensor')
                if c in e]
        print(f'  {k:<12}' + ' '.join(f'{c} {e[c]:.1e}' for c in keys))
        for c in keys:
            assert e[c] < TOL[c], (label, k, c, e[c])
    return twins


# ------------------------------------------------------------------------------------------------------------ the pinned states

def test_free_model_has_no_constraints():
    for name in ss.DEFAULT_MODELS:
        full = ss.base_model(name)
        m = model(name)
        assert m.npair == m.c.npair == len(m.pair_geom1) == 0 and not m.jnt_limited.any()
        assert full.npair > 0 and full.jnt_limited.any() and full.npair == len(full.pair_geom1)     # the copy left the model alone
        on, off = fluid_models(name)
        assert off.opt_density == off.opt_viscosity == 0 and on.opt_density == m.opt_density > 0 and on.opt_viscosity > 0
        assert not on.jnt_stiffness.any() and not on.dof_damping.any() and m.dof_damping.any()


@pytest.mark.parametrize('name', ss.MODELS)
def test_smooth_states_keep_their_properties(name):
    """each pinned state still reaches its edge, and nefc = 0 on the oracle's side of the free model"""
    m = model(name)
    names = ss.state_names(m)
    assert 'quat_a' in names and len(names) >= (7 if name == 'ball' else 11), names
    p = {k: ss.describe(m, k) for k in names}
    for k in names:
        assert p[k]['range_reach'] > 0.85, (k, p[k])        # a hinge near the end of its range
        assert p[k]['min_act'] > 0, (k, p[k])                # every activation nonzero
        assert oracle(name)[k]['nefc'] == 0, k
    assert abs(p['quat_w0']['quat_w']) < 1e-3 and abs(p['quat_a']['quat_w']) > 0.3
    assert p['quat_neg']['quat_w'] == -p['quat_a']['quat_w']
    assert abs(p['quat_half']['quat_norm'] - 0.5) < 1e-6 and abs(p['quat_double']['quat_norm'] - 2) < 1e-6
    if 'far_1e3' in names:
        assert 100 <= p['far_1e2']['root_xy'] < 500 <= p['far_1e3']['root_xy'] < 1000, (p['far_1e2'], p['far_1e3'])
    if 'wings_only' in names:
        assert p['wings_only']['wing_speed'] > 1000 and p['wings_only'].get('linvel', 0) == 0
    if 'body_only' in names:
        b = p['body_only']
        assert b['hinge_speed'] == 0 and abs(b['linvel'] - ss.TERMINAL_LINVEL) < 1e-3 and abs(b['angvel'] - ss.TERMINAL_ANGVEL) < 1e-2
    if 'flight' in names:
        f = p['flight']
        assert f['wing_speed'] > 1000 and f['linvel'] > 0.99 * ss.TERMINAL_LINVEL and f['angvel'] > 0.99 * ss.TERMINAL_ANGVEL


def test_wing_beat_speeds_are_real_flight_speeds():
    """the wing speeds come from the flight task's wing-beat table at 218 Hz: of order 1e3 rad/s, over about +-1 rad"""
    peak = max(np.abs(ss.wing_beat(r)[1]).max() for r in range(23))
    assert 1000 < peak < 3000, peak


# ----------------------------------------------------------------------------------------------------------- host emulation

@pytest.fixture(scope='module')
def emu():
    ge.build()
    return ge.EMU


@pytest.mark.parametrize('name', ss.MODELS)
def test_smooth_gates_under_emulation(emu, name):
    """the kernel source on the host: every state of the model as one env of a batch"""
    m = model(name)
    gate(f'emulation {name}', name, st.BatchedStepper(m, len(ss.state_names(m)), lib_path=emu), m)


@pytest.mark.parametrize('name', ss.MODELS)
def test_fluid_gates_under_emulation(emu, name):
    m_on, m_off = fluid_models(name)
    n = len(ss.state_names(m_on))
    fluid_gate(f'emulation fluid {name}', name, (st.BatchedStepper(m_on, n, lib_path=emu), st.BatchedStepper(m_off, n, lib_path=emu)))


@pytest.mark.parametrize('name', ss.DEFAULT_MODELS)
def test_sign_scale_and_translation_twins_under_emulation(emu, name):
    m = model(name)
    gate_twins(f'emulation {name}', m, st.BatchedStepper(m, len(ss.state_names(m)), lib_path=emu))


@pytest.mark.parametrize('name', ss.DEFAULT_MODELS)
def test_default_models_carry_over_under_emulation(emu, name):
    """the shipped models, with their contact pairs and joint limits: the fields before the constraint stage hold the same gates in
    a batch where some envs have constraint rows and some have none"""
    m = model(name, free=False)
    sim = st.BatchedStepper(m, len(ss.state_names(m)), lib_path=emu)
    gate(f'emulation {name} with contacts', name, sim, m, keys=PRE_CONSTRAINT, free=False)
    nefc = sim.get(st.NEFC)[:, 0]
    assert nefc.max() > 0, nefc


def test_world_subtree_com_is_the_whole_scene(emu):
    """fb_get(SUBTREE_COM) of the world body is the centre of mass of every body (MuJoCo subtree_com[0]); it read back the reference
    point, because the kernels keep no composite inertia for the world"""
    for name in ('walk', 'ball'):
        m = model(name)
        sim = st.BatchedStepper(m, 1, lib_path=emu)
        d = ss.device_fields(m, sim, ['far_1e3' if name == 'walk' else 'quat_a'], [0], step=False)[0]
        o = oracle(name)['far_1e3' if name == 'walk' else 'quat_a']
        c = o['subtree_com'].reshape(-1, 3)
        assert np.abs(d['subtree_com'].reshape(-1, 3)[0] - c[0]).max() < 1e-4 * max(1.0, np.abs(c[0]).max()), (name, c[0])


def test_observation_program_refuses_the_world_subtree_com(emu):
    m = model('walk')
    sim = st.BatchedStepper(m, 1, lib_path=emu)
    with pytest.raises(st.StepperError, match='subtree_com body id'):
        sim.obs_program([(st.OBS_SUBTREE_COM, 0, 3)], [], m.body_id('walker/thorax'), 1)
    assert sim.obs_program([(st.OBS_SUBTREE_COM, m.body_id('walker/thorax'), 3)], [], m.body_id('walker/thorax'), 1) == 3


# ----------------------------------------------------------------------------------------------------------------- on the H100

@pytest.mark.gpu
@pytest.mark.parametrize('blob', ['0', '1'])
@pytest.mark.parametrize('name', GPU_MODELS)
def test_smooth_gates_on_gpu(name, blob, monkeypatch):
    """every state as one env of a batch, the sweep program copied into shared memory per CTA (FB_BLOB = 1) and read in place (0)"""
    monkeypatch.setenv('FB_BLOB', blob)
    m = model(name)
    gate(f'H100 {name} FB_BLOB={blob}', name, st.BatchedStepper(m, len(ss.state_names(m))), m)


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['walk', 'flight', 'ball'])
def test_smooth_gates_on_gpu_4096_envs(name):
    """the configuration bench.py times: 4096 envs, sweep program read in place.  Env i holds state (i // 4 + i) mod S, so every CTA
    of 4 warps holds 4 different states and every state runs at every warp position many times over."""
    m = model(name)
    n, S = 4096, len(ss.state_names(m))
    assign = [(i // 4 + i) % S for i in range(n)]
    assert len({(a, i % 4) for i, a in enumerate(assign)}) == 4 * S
    gate(f'H100 {name} 4096 envs', name, st.BatchedStepper(m, n), m, assign=assign)


@pytest.mark.gpu
@pytest.mark.parametrize('name', ss.DEFAULT_MODELS)
def test_fluid_gates_on_gpu(name):
    m_on, m_off = fluid_models(name)
    n = len(ss.state_names(m_on))
    fluid_gate(f'H100 fluid {name}', name, (st.BatchedStepper(m_on, n), st.BatchedStepper(m_off, n)))


@pytest.mark.gpu
@pytest.mark.parametrize('name', ss.DEFAULT_MODELS)
def test_sign_scale_and_translation_twins_on_gpu(name):
    m = model(name)
    gate_twins(f'H100 {name}', m, st.BatchedStepper(m, len(ss.state_names(m))))


@pytest.mark.gpu
@pytest.mark.parametrize('name', ss.DEFAULT_MODELS)
def test_default_models_carry_over_on_gpu(name):
    """the shipped models in a 256-env batch: the pinned states, each at every warp position, among envs with contacts and limits"""
    m = model(name, free=False)
    S = len(ss.state_names(m))
    assign = [(i // 4 + i) % S for i in range(256)]
    sim = st.BatchedStepper(m, 256)
    gate(f'H100 {name} with contacts', name, sim, m, assign=assign, keys=PRE_CONSTRAINT, free=False)
    assert sim.get(st.NEFC)[:, 0].max() > 0
