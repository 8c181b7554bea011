"""The finish kernel (fb_constraint.h kfin_f1 .. kfin_f10) against fp64 restatements, per element (tests/finish_states.py): the solver's
forces into qacc (the Z^T f path) and into qfrc_constraint (the J^T f path), the contact wrenches and delta accelerations behind the
accelerometer and force sensors, the touch ray test, and the semi-implicit Euler step of hinge, free and ball joints and of the filter
activations.  The states are the 14 pinned solver states (nefc 1 - 105, register and generic solve paths), pinned cases on model
copies that reach the touch branches those never do, and the ball model with the claws on the moving ball (tier 2 through the
oracle's free-joint surrogate); the placements are those of tests/test_solver_gates.py.

Tier 1 (the kernel on the device's own inputs, so that solver and collision error drop out; tolerance = measured x 2.5):
  qfrc_constraint   per dof |dq_i| / sqrt(M_ii) against fp64 J^T f_dev, relative to the largest dof          qfrc_constraint
  qacc              backward against the device's M and qfrc_smooth + qfrc_constraint, forward against the  qacc_back, qacc_fwd
                    fp64 solve of the same numbers (smooth_states.solve_errors): the Z^T f and J^T f paths agree
  dqvel / h         forward against the fp64 solve of M + h diag(damping), the same right-hand side          dv_fwd
  qpos, act, time   fp64 Euler step from the device's qpos0, its qvel after the step, act0 + h (clamp(ctrl) -   qpos_ulps, act_ulps,
                    act0) / tau; in fp32 ulps (quaternions: q (x) exp(w h / 2), body frame, normalised)        time (exact)
  accelerometer,    per sensor |ds| / (max |s| + parity_common.SENSOR_FLOOR) against                          accelerometer, force
  force             sensor_fd_reference.inverse_sensors at (qacc_dev, efc_force_dev)
  touch             per sensor |ds| / (|s| + 1e-3) against the fp64 ray test on the device's contacts, forces   touch
                    and site poses; a sensor with a positive-force contact within TOUCH_BAND of its site's surface
                    is counted and printed, not gated
Tier 2 (end to end against the oracle's forward() and one step; tolerances admit the solver's error, test_solver_gates.py): the same
fields, prefixed t2_.

The touch band is measured (band_sweep, test_touch_band_is_measured_*): on the states whose positive-force contacts pass outside a
site, each site's radius is set so that the fp64 ray of its nearest contact passes at +-1e-3 .. +-1e-7 radii of the surface, and the
kernel's touch is compared with the fp64 ray test.  They part only within 1.4e-7 radii under emulation and 1.0e-6 radii on the H100
(its fused multiply-adds), never at 1e-5 or more.  TOUCH_BAND = 1e-3 radii holds the measurement with three decades to spare, and the
gate asserts the measured edge stays below 0.1 of it.  No pinned contact lies in the band: the smallest |margin| of a positive-force contact is 4.3e-2 radii
(test_touch_band_holds_no_pinned_contact).
"""
import hashlib

import numpy as np
import pytest

import __graft_entry__ as ge
import finish_states as fs
import smooth_states as sms
import solver_states as ss
from flybody_b200 import stepper as st
from flybody_b200.flymodel import load_model

# measured under emulation (the kernel source on the host) and on an H100 (80 GB HBM3, 700 W power limit), the larger of the two x 2.5;
# the worst state of the larger in parentheses
TOL = dict(
    qfrc_constraint=1.7e-5,      # emulation 6.6e-6 (condim13), H100 4.5e-6
    qacc_back=1.7e-5,            # emulation 6.7e-6 (rows64), H100 6.3e-6
    qacc_fwd=1.5e-6,             # H100 5.9e-7 (middle_mu1_a), emulation 5.0e-7
    dv_fwd=8e-7,                 # H100 3.2e-7 (smooth states, walk_jf0), emulation 2.5e-7; contact states 1.9e-7 / 1.5e-7
    qpos_ulps=5.3,               # H100 2.09 (condim13), emulation 2.0 (smooth states, walk_wings)
    act_ulps=5.2,                # emulation and H100 2.07 (smooth states, walk_wings)
    time=0.0,                    # exact: fp32(time0 + fp32(h))
    accelerometer=3e-7,          # emulation and H100 1.2e-7 (zones_generic)
    force=2.2e-5,                # emulation 8.5e-6 (geom1_inside), H100 6.3e-6
    touch=1.1e-7,                # H100 4.2e-8 (geom1_inside), emulation 3.6e-8
    inverse_touch=1e-7,          # emulation 4.0e-8 (condim13), H100 3.5e-8
    inverse_force=2.2e-5,        # emulation 8.5e-6 (middle_mu1_b), H100 6.2e-6
    # tier 2: the solver's per-contact error (test_solver_gates.py PER_MAX) carried through
    t2_qfrc_constraint=1.2e-3,   # H100 4.6e-4 (middle_mu1_b, noslip 0), emulation 3.7e-4
    t2_qacc=1e-3,                # H100 3.9e-4 (middle_mu1_b, noslip 0), emulation 2.3e-4
    t2_dqvel=1.1e-3,             # H100 4.1e-4 (middle_mu1_b, noslip 0), emulation 2.3e-4
    t2_qpos=2.3e-5,              # H100 9.0e-6 (middle_mu1_b), emulation 7.3e-6; cm / rad
    t2_accelerometer=2.8e-4,     # emulation and H100 1.1e-4 (geom1_inside)
    t2_force=8.7e-3,             # H100 3.5e-3 (middle_mu1_b), emulation 2.6e-3
    t2_touch=6.3e-3,             # H100 2.5e-3 (middle_mu1_b), emulation 1.9e-3
)
NAMES = list(fs.all_states())
DEVICE_OUTPUTS = ('qM', 'qfrc_smooth', 'qfrc_constraint', 'qacc', 'force', 'con', 'site_xpos', 'site_xmat', 'sensordata', 'qpos1',
                  'qvel1', 'act1')

_ORACLE = {}


def oracle(name, noslip=None):
    key = (name, noslip)
    if key not in _ORACLE:
        mk, t = fs.all_states()[name]
        m = fs.MODELS[mk](noslip)
        _ORACLE[key] = fs.oracle_stage(m, fs.state_inputs(m, mk, t))
    return _ORACLE[key]


def run(label, make_sim, noslip=None, n_envs=None, names=None):
    """every pinned state on its model (one batch per model, one env per state; with n_envs, env i holds state (i // 4 + i mod 4) mod S
    of that model's S states, so every state runs at every warp position of a 4-warp CTA), gated and printed one row per state (its
    worst env)"""
    names = names or NAMES
    by_model = {}
    for k in names:
        by_model.setdefault(fs.all_states()[k][0], []).append(k)
    worst, bad = {}, []
    for mk, ks in by_model.items():
        m = fs.MODELS[mk](noslip)
        n = n_envs or len(ks)
        assign = [(i // 4 + i % 4) % len(ks) for i in range(n)] if n_envs else list(range(n))
        assert n_envs is None or len({(a, i % 4) for i, a in enumerate(assign)}) == 4 * len(ks)
        inputs = [fs.state_inputs(m, mk, fs.all_states()[k][1]) for k in ks]
        dev = fs.device_step(m, make_sim(m, n), [inputs[a] for a in assign])
        seen = {}
        for i, d in enumerate(dev):
            k = ks[assign[i]]
            assert d['flags'] == 0, (label, k, i, d['flags'])
            # envs of one state whose outputs are bitwise equal have equal errors: restate each distinct result once
            key = (k, hashlib.sha1(b''.join(np.ascontiguousarray(d[c]).tobytes() for c in DEVICE_OUTPUTS)).hexdigest())
            if key not in seen:
                seen[key] = fs.errors(m, d, oracle(k, noslip))
            e = seen[key]
            w = worst.setdefault(k, dict(nefc=d['nefc']))
            for c, v in e.items():
                w[c] = max(w.get(c, 0.0), v)
                if c in TOL and not v <= TOL[c]:
                    bad.append((k, i, c, v))
    cols = [c for c in TOL if any(c in w for w in worst.values())] + ['band']
    print(f'\n{label}')
    print('  ' + f'{"state":<14}{"nefc":>5}' + ''.join(f'{c.replace("t2_", "2:")[:10]:>11}' for c in cols))
    for k in names:
        w = worst[k]
        print('  ' + f'{k:<14}{w["nefc"]:>5}' + ''.join(f'{w.get(c, float("nan")):11.2e}' for c in cols))
    assert not bad, (label, bad[:8])
    return worst


EULER_KEYS = ('qpos_ulps', 'act_ulps', 'time', 'dv_fwd', 'qacc_fwd')


def integration_gate(label, name, make_sim):
    """tier 1's Euler gates (qpos, act, time, one substep's dqvel / h) on every smooth_states state of model `name`: hinges over their
    whole range, quaternions at -q, 0.5 q, 2 q and a 180-degree turn, the root 1e3 cm out, wing-beat and termination speeds, ball
    joints; the constraint-free copy, so no oracle is needed.  One row per state"""
    m = sms.free_model(sms.base_model(name))
    names = sms.state_names(m)
    ins = [sms.state_inputs(m, k) for k in names]
    dev = fs.device_step(m, make_sim(m, len(names)), [(q, v, c) for q, v, _, c in ins],
                         act=np.array([a for _, _, a, _ in ins]) if m.na else None)
    rows = {}
    for k, d in zip(names, dev):
        assert d['flags'] == 0, (label, name, k)
        e = fs.errors(m, d)
        rows[k] = {c: e[c] for c in EULER_KEYS if c in e}
    print(f'\n{label} {name}: Euler step of the smooth states')
    print('  ' + f'{"state":<12}' + ''.join(f'{c:>11}' for c in EULER_KEYS))
    for k, w in rows.items():
        print('  ' + f'{k:<12}' + ''.join(f'{w.get(c, float("nan")):11.2e}' for c in EULER_KEYS))
    bad = [(k, c, v) for k, w in rows.items() for c, v in w.items() if not v <= TOL[c]]
    assert not bad, (label, name, bad)
    return rows


def inverse_gate(label, lib):
    """fb_inverse's sensor pass (kinv_sensors: a copy of kfin_f9's touch and force code) at the device's forward qacc, against the
    same restatements on its own contacts and forces: touch by the fp64 ray test on the inverse's contact rows and the forward
    stage's site poses, force by sensor_fd_reference.inverse_sensors at (qacc, the inverse's contact forces)"""
    from flybody_b200.inverse_dynamics import inverse
    from parity_common import SENSOR_FLOOR
    worst = {}
    for k, (mk, t) in fs.all_states().items():
        if mk == 'flight':
            continue
        m = fs.MODELS[mk]()
        x = fs.state_inputs(m, mk, t)
        sim = st.BatchedStepper(m, 1, lib_path=lib) if lib else st.BatchedStepper(m, 1)
        d = fs.device_step(m, sim, [x])[0]
        sim.close()
        r = inverse(m, x[0], x[1], d['qacc'], lib_path=lib, sensors=True)
        o = oracle(k)
        c, rows = r.contacts, o['con'][o['con'][:, 12] >= 0]          # the inverse lists the contacts that have rows
        assert np.array_equal(c.geom, rows[:, 7:9].astype(np.int64)), (label, k)          # the forward's contacts, in order
        con, f = np.zeros((len(rows), 16)), np.zeros(o['nefc'])
        for i, row in enumerate(rows):
            adr, dim = int(row[12]), (3 if row[9] >= 3 else 1)
            con[i, 1:4], con[i, 4:7], con[i, 7:10], con[i, 12] = c.pos[i], c.normal[i], row[7:10], adr
            f[adr:adr + dim] = c.force[i][:dim]
        sens = np.asarray(r.sensordata).reshape(-1)
        tr = fs.touch_reference(m, con, f, d['site_xpos'], d['site_xmat'])
        touch, band = fs.touch_error(m, sens, tr, SENSOR_FLOOR[fs.TOUCH])
        force = fs.acc_sensor_errors(m, sens, fs.sensor_restatement(o, d['qacc'], f), SENSOR_FLOOR)[1]
        worst[k] = dict(touch=touch, force=force, band=band)
    print(f'\n{label}: fb_inverse sensors at the forward qacc')
    for k, w in worst.items():
        print(f'  {k:<14} touch {w["touch"]:9.2e}  force {w["force"]:9.2e}  band {w["band"]}')
    bad = [(k, w) for k, w in worst.items() if not (w['touch'] <= TOL['inverse_touch'] and w['force'] <= TOL['inverse_force'])]
    assert not bad, (label, bad[:5])
    return worst


# the states whose positive-force contacts pass outside a site at margins of -0.7 .. 9 radii (the walk states' outside contacts are
# floor contacts at the claw's tip whose rays run up the site's axis, margin -1)
BAND_STATES = ('miss_one', 'miss_rows64', 'geom1_outside', 'geom1_miss')
BAND_MARGINS = (1e-3, 1e-4, 1e-5, 1e-6, 1e-7)


def band_sweep(label, make_sim):
    """measure how close to a touch site's surface the kernel's fp32 hit decision and the fp64 ray test part.  For each state of
    BAND_STATES, every touch site with a positive-force contact outside it gets the radius (in fp32) at which the fp64 ray of its
    nearest such contact passes at margin +-delta of the surface (the contacts and the dynamics do not depend on the radius); one
    step per (state, delta), and per sensor the device's touch against the fp64 ray test.  Returns the largest |margin| (site
    radii) of a sensor's nearest positive-force contact where the two disagree, and the number of (sensor, delta) cases"""
    from parity_common import SENSOR_FLOOR
    worst, cases, flips = 0.0, 0, []
    for k in BAND_STATES:
        mk, t = fs.all_states()[k]
        m0 = fs.MODELS[mk]()
        x = fs.state_inputs(m0, mk, t)
        d0 = fs.device_step(m0, make_sim(m0, 1), [x])[0]
        target = {}
        for site in fs.touch_sites(m0):
            cs = [c for c in fs.touch_contacts(m0, site, d0['con'], d0['force'], d0['site_xpos'], d0['site_xmat'])
                  if c['fn'] > 0 and not c['inside'] and -0.7 < c['margin'] < 9.0]
            if cs:
                target[site] = min(cs, key=lambda c: abs(c['margin']))['margin'] + 1.0      # distance / radius, at the shipped radius
        for delta in BAND_MARGINS:
            for sign in (1.0, -1.0):
                radii = {site: float(np.float32(D * float(m0.site_size[site, 0]) / (1.0 + sign * delta))) for site, D in target.items()}
                m = fs.site_radius_model(m0, radii)
                d = fs.device_step(m, make_sim(m, 1), [x])[0]
                assert np.array_equal(d['force'], d0['force']) and np.array_equal(d['con'], d0['con']), (label, k)
                for s in range(m.nsensor):
                    site = int(m.sensor_objid[s])
                    if site not in target:
                        continue
                    cases += 1
                    cs = [c for c in fs.touch_contacts(m, site, d['con'], d['force'], d['site_xpos'], d['site_xmat']) if c['fn'] > 0]
                    ref = sum(c['fn'] for c in cs if c['hit'])
                    got = d['sensordata'][int(m.sensor_adr[s])]
                    if abs(got - ref) > 1e-3 * (abs(ref) + SENSOR_FLOOR[fs.TOUCH]):
                        near = min(abs(c['margin']) for c in cs)
                        worst = max(worst, near)
                        flips.append((k, s, sign * delta, near))
    print(f'\n{label}: touch decisions at margins +-{BAND_MARGINS} site radii, {cases} (sensor, margin) cases; '
          f'{len(flips)} disagree with fp64, the largest |margin| of one {worst:.2e} (band {fs.TOUCH_BAND:.0e})')
    for f in flips:
        print('  ', f)
    return worst, cases


# ------------------------------------------------------------------------------------------------------------ the pinned states

def test_finish_states_keep_their_properties():
    """the pinned states reach every branch of the touch ray test (a positive-force miss, the site body as geom1 inside, outside with
    a hit and missing, a zero-force contact, a point inside the site, outside with a hit), nefc <= 32 and > 32, limits only, and the
    claws pressing on the moving ball (the ball as geom1) on both solve paths"""
    reach = {}
    for k, (mk, t) in fs.all_states().items():
        m = fs.MODELS[mk]()
        o = oracle(k)
        reach[k] = br = fs.touch_branches(m, o['con'], o['force'], o['site_xpos'], o['site_xmat'])
        g1 = [c for s in fs.touch_sites(m) for c in fs.touch_contacts(m, s, o['con'], o['force'], o['site_xpos'], o['site_xmat'])
              if c['side'] == 1 and c['fn'] > 0]
        br['geom1_inside'] = sum(c['inside'] for c in g1)
        br['geom1_outside_hit'] = sum(c['hit'] and not c['inside'] for c in g1)
        br['geom1_miss'] = sum(not c['hit'] for c in g1)
        br['nefc'], br['ncon'] = o['nefc'], o['ncon']
        ball = [g for g in range(m.ngeom) if mk == 'ball' and int(m.geom_bodyid[g]) == 1]
        br['ball_geom1'] = sum(1 for r in o['con'] if r[12] >= 0 and int(r[7]) in ball and o['force'][int(r[12])] > 0)
        print(k, br)
    assert reach['miss_one']['miss'] >= 1 and reach['miss_one']['nefc'] <= ss.FB_SOLVE_NCAP
    assert reach['miss_rows64']['miss'] >= 1 and reach['miss_rows64']['nefc'] > ss.FB_SOLVE_NCAP
    assert reach['geom1_inside']['geom1_inside'] >= 1
    assert reach['geom1_outside']['geom1_outside_hit'] >= 1
    assert reach['geom1_miss']['geom1_miss'] >= 1
    assert reach['flight_limits']['ncon'] == 0 < reach['flight_limits']['nefc']
    # the ball states: the ball geom as geom1 of positive-force claw contacts, on both solve paths, the claws' touch sensors reached
    for k in ('ball_rest', 'ball_few', 'ball_many'):
        assert reach[k]['ball_geom1'] >= 2 and reach[k]['inside'] + reach[k]['outside_hit'] >= 1, (k, reach[k])
    assert reach['ball_few']['nefc'] <= ss.FB_SOLVE_NCAP < reach['ball_many']['nefc']
    solver = [reach[k] for k in ss.STATES]
    assert sum(r['zero_force'] for r in solver) > 0 and sum(r['inside'] for r in solver) > 0
    assert sum(r['outside_hit'] for r in solver) > 0
    # the solver states alone never miss and never have the site body as geom1: the reason for the extra states
    assert sum(r['miss'] + r['geom1'] for r in solver) == 0


def test_touch_band_holds_no_pinned_contact():
    """the smallest |margin| (in site radii) of a positive-force contact on a touch body over the pinned states is far outside the
    band, so every touch sensor of every state is gated"""
    smallest = np.inf
    for k, (mk, _) in fs.all_states().items():
        m, o = fs.MODELS[mk](), oracle(k)
        for s in fs.touch_sites(m):
            for c in fs.touch_contacts(m, s, o['con'], o['force'], o['site_xpos'], o['site_xmat']):
                if c['fn'] > 0:
                    smallest = min(smallest, abs(c['margin']))
    print(f'\nsmallest |margin| of a positive-force touch contact: {smallest:.2e} site radii (band {fs.TOUCH_BAND:.0e})')
    assert smallest > 10 * fs.TOUCH_BAND


def test_touch_sites_the_ray_test_does_not_know_are_refused(emu):
    """kfin_f9, kinv_sensors and orc_sensors_acc ray-test a capsule site and treat any other as a sphere: an ellipsoid, box or
    cylinder touch site is refused by fb_create and orc_create instead of being tested against the wrong shape"""
    from oracle import fly_oracle as fo
    m = load_model('walk')
    for t in (4, 5, 6):                     # ellipsoid, cylinder, box
        bad = m.copy()
        tp = bad.site_type.copy()
        tp[fs.touch_sites(m)[2]] = t
        bad.a['site_type'] = tp
        bad = bad.rebuild()
        with pytest.raises(st.StepperError, match=f'touch site of type {t}'):
            st.BatchedStepper(bad, 2, lib_path=emu)
        with pytest.raises(ValueError, match='orc_create refused'):
            fo.Oracle(bad)
    ok = m.copy()
    tp = ok.site_type.copy()
    tp[fs.touch_sites(m)] = fs.SPHERE
    ok.a['site_type'] = tp
    ok = ok.rebuild()
    st.BatchedStepper(ok, 2, lib_path=emu).close()        # a sphere touch site is accepted by both
    fo.Oracle(ok)


def test_applied_forces_stay_out_of_the_force_sensors(emu):
    """the documented deviation (include/flybody_b200.h, fb_inverse.h): xfrc_applied moves qacc but does not enter cfrc_int, so the
    force sensor of the body that carries the wrench reads what the xfrc-free restatement gives at the same qacc, not that plus the
    wrench.  Pinned: changing it must be deliberate"""
    from parity_common import SENSOR_FLOOR
    from sensor_fd_reference import FORCE
    m = fs.walk_model()
    x = ss.state_inputs(m, *ss.STATES['one_contact'][0])
    sim = st.BatchedStepper(m, 1, lib_path=emu)
    s = [k for k in range(m.nsensor) if m.sensor_type[k] == FORCE][0]
    site, adr = int(m.sensor_objid[s]), int(m.sensor_adr[s])
    b = int(m.site_bodyid[site])
    F = np.array([0.0, 0.0, 0.5])
    xf = np.zeros((m.nbody, 6))
    xf[b, :3] = F
    d = fs.device_step(m, sim, [x], xfrc=xf[None])[0]
    o = oracle('one_contact')
    ref = fs.sensor_restatement(o, d['qacc'], d['force'])[adr:adr + 3]     # the restatement without xfrc_applied
    scale = np.abs(ref).max() + SENSOR_FLOOR[FORCE]
    err = float(np.abs(d['sensordata'][adr:adr + 3] - ref).max() / scale)
    shown = float(np.abs(d['site_xmat'].reshape(-1, 3, 3)[site].T @ F).max() / scale)     # what the wrench would add to the reading
    moved = float(np.abs(d['qacc'] - o['qacc']).max() / np.abs(o['qacc']).max())
    print(f'\nxfrc_applied {F[2]} on body {b}: qacc moves by {moved:.2e} (relative); its force sensor against the xfrc-free restatement '
          f'{err:.2e}, with the wrench it would be off by {shown:.2e}; the error is {err * scale / F[2]:.1e} of the wrench')
    # emulation 9.1e-7 against the force gate's 2.2e-5, while the wrench would move the reading by 1.4e-1
    assert moved > 1e-2 and err <= TOL['force'] and shown > 1000 * TOL['force']


# ----------------------------------------------------------------------------------------------------------- host emulation

@pytest.fixture(scope='module')
def emu():
    ge.build()
    return ge.EMU


@pytest.fixture(scope='module')
def emu_chol(tmp_path_factory):
    return ss.build_chol_variants(tmp_path_factory.mktemp('emu_chol'), ge.CSRC)


@pytest.mark.parametrize('placement', ['default', 'ncap0', 'chol_reg0', 'chol_reg8', 'noslip0', 'noslip10'])
def test_finish_gates_under_emulation(emu, emu_chol, placement, monkeypatch):
    """the kernel source on the host: the register path (default), the generic path for every nefc (FB_SOLVE_NCAP = 0), the
    record-side Hessian factorisation above 0 / 8 columns, and noslip off and with 10 sweeps (the qacc of the Z^T f path after noslip)"""
    lib, noslip = emu, None
    if placement == 'ncap0':
        monkeypatch.setenv('FB_SOLVE_NCAP', '0')
    elif placement.startswith('chol_reg'):
        lib = emu_chol[int(placement[-1])]
    elif placement.startswith('noslip'):
        noslip = int(placement[6:])
    run(f'emulation {placement}', lambda m, n: st.BatchedStepper(m, n, lib_path=lib), noslip=noslip)


@pytest.mark.parametrize('name', sms.MODELS)
def test_euler_step_of_the_smooth_states_under_emulation(emu, name):
    integration_gate('emulation', name, lambda m, n: st.BatchedStepper(m, n, lib_path=emu))


def test_inverse_touch_and_force_under_emulation(emu):
    inverse_gate('emulation', emu)


def test_touch_band_is_measured_under_emulation(emu):
    worst, cases = band_sweep('emulation', lambda m, n: st.BatchedStepper(m, n, lib_path=emu))
    assert cases >= 100 and worst < 0.1 * fs.TOUCH_BAND


# ----------------------------------------------------------------------------------------------------------------- on the H100

@pytest.mark.gpu
@pytest.mark.parametrize('placement', ['blob1', 'blob0', 'ncap0'])
def test_finish_gates_on_gpu(placement, monkeypatch):
    """every state as one env of its model's batch, the sweep program in shared memory (FB_BLOB = 1), read in place (0), and the
    generic solve path for every nefc (FB_SOLVE_NCAP = 0)"""
    if placement == 'ncap0':
        monkeypatch.setenv('FB_SOLVE_NCAP', '0')
    else:
        monkeypatch.setenv('FB_BLOB', placement[-1])
    run(f'H100 {placement}', lambda m, n: st.BatchedStepper(m, n))


@pytest.mark.gpu
def test_finish_gates_on_gpu_4096_envs():
    """the configuration bench.py times: 4096 envs per model; env i holds state (i // 4 + i mod 4) mod S, so every state runs at every
    warp position of a 4-warp CTA"""
    run('H100 4096 envs', lambda m, n: st.BatchedStepper(m, n), n_envs=4096)


@pytest.mark.gpu
@pytest.mark.parametrize('noslip', [0, 10])
def test_finish_gates_noslip_on_gpu(noslip):
    run(f'H100 noslip {noslip}', lambda m, n: st.BatchedStepper(m, n), noslip=noslip)


@pytest.mark.gpu
@pytest.mark.parametrize('name', sms.MODELS)
def test_euler_step_of_the_smooth_states_on_gpu(name):
    integration_gate('H100', name, lambda m, n: st.BatchedStepper(m, n))


@pytest.mark.gpu
def test_touch_band_is_measured_on_gpu():
    worst, cases = band_sweep('H100', lambda m, n: st.BatchedStepper(m, n))
    assert cases >= 100 and worst < 0.1 * fs.TOUCH_BAND


@pytest.mark.gpu
def test_inverse_touch_and_force_on_gpu():
    inverse_gate('H100', None)
