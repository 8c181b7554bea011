"""The constraint solve against the fp64 oracle, contact by contact, on the analytic-contact walk model (tests/solver_states.py), at
the solver's edges (nefc 1 - 105, the 32 / 33 handover of the register path, Hessian blocks of 24 / 25 columns, all three cone zones,
condim 1 and 3) and through every placement of the solve: the register and generic paths, the shared-memory and record Hessian
factorisations, the shared-memory and global-memory sweep programs, mixed batches, noslip off / on, and across substeps.

Gates (fp32 stepper vs fp64 oracle; tolerance = measured x 2.5, the measurement is printed):
  max |df| / max |f|                                     over a state's rows                            MAXREL
  per contact max_rows |df| / (|f_n| + 1e-4 max |f|),
  per limit row |df| / (|f| + 1e-4 max |f|)              90th percentile over the placement's contacts  PER_P90
                                                         worst contact                                   PER_MAX
  per row |df_r| / (2^-24 jar_resolution_r)              worst row (fp32 resolution of the row's jar)   RES_ULPS
  cone zone of every contact from the forces             equal, outside a 1e-2 band at zone boundaries
  cone feasibility of the device forces                  |f_t / mu| <= f_n (1 + 1e-5)
  nefc, ncon, the contact pairs                          identical; FLAGS 0

PER_MAX is loose because of two light middle-zone contacts (middle_mu1_a / _b): their forces are 1e-3 - 1e-2 of the state's largest
force, and the terms that cancel in their jar are 1e4 times larger than their force (solver_states.jar_resolution).  Their error does
not move with the fp32 rounding of the model (solver_states.fp32_model: 5.60e-3 -> 5.44e-3, 1.87e-3 -> 1.87e-3), and it is 11 - 13
units of 2^-24 of those terms, like the other rows' (up to 37): RES_ULPS holds them at that resolution.
"""
import numpy as np
import pytest

import __graft_entry__ as ge
import solver_states as ss
from flybody_b200 import stepper as st
from flybody_b200.flymodel import load_model
from oracle import fly_oracle as fo
from parity_common import reset_qpos, sensor_mean_error

# measured under emulation (the kernel source on the host) and on an H100 (80 GB HBM3, 700 W), the larger of the two x 2.5
MAXREL = 3.2e-4           # H100 1.29e-4 (rows105, noslip off), emulation 1.24e-4
PER_P90 = 1.9e-4          # H100 7.6e-5, emulation 6.5e-5
PER_MAX = 1.4e-2          # emulation 5.6e-3 (middle_mu1_a), H100 2.5e-3 (middle_mu1_b)
RES_ULPS = 300            # H100 121 units of 2^-24 (rows105), emulation 37; the two middle_mu1 states: 11 and 13 under emulation
NAMES = list(ss.STATES)
TRIPLES = [ss.STATES[k][0] for k in NAMES]

_ORACLE = {}


def model(noslip=None):
    return ss.analytic_model(load_model('walk'), noslip=noslip)


def oracle(noslip=None):
    """oracle solutions and jar resolutions of every targeted state, per noslip setting (cached: the oracle is deterministic)"""
    if noslip not in _ORACLE:
        m = model(noslip)
        _ORACLE[noslip] = [(ss.oracle_solution(m, *t), ss.jar_resolution(m, *t)) for t in TRIPLES]
    return _ORACLE[noslip]


def gate(label, sim, m, noslip=None, assign=None):
    """run the targeted states on `sim` (env i holds state assign[i]; default: one env per state), gate every env against the oracle
    and print one row per state"""
    assign = list(range(len(NAMES))) if assign is None else assign
    ora = oracle(noslip)
    dev = ss.device_solutions(m, sim, TRIPLES, assign)
    per, worst, bad = [], {}, []
    for i, d in enumerate(dev):
        k = assign[i]
        o, res = ora[k]
        assert d['flags'] == 0, (label, NAMES[k], i, d['flags'])
        assert (d['nefc'], d['ncon']) == (o['nefc'], o['ncon']), (label, NAMES[k], i, d['nefc'], o['nefc'], d['ncon'], o['ncon'])
        assert np.array_equal(d['con'][:, 7:10], o['con'][:, 7:10]), (label, NAMES[k], i)          # same pairs, same condim
        assert np.array_equal(d['con'][:, 12], o['con'][:, 12]), (label, NAMES[k], i)               # same row addresses
        e = ss.errors(d, o, m.opt_impratio)
        e['res'] = float((np.abs(d['force'] - o['force']) / (res + 1e-30)).max()) * 2.0 ** 24 if o['nefc'] else 0.0
        if not (e['maxrel'] < MAXREL and e['per'] < PER_MAX and e['res'] < RES_ULPS and e['cone'] <= ss.CONE_SLACK
                and not e['zone_mismatch']):
            bad.append((NAMES[k], i, {key: e[key] for key in ('maxrel', 'per', 'res', 'cone', 'zone_mismatch')}))
        per += e['per_all']
        w = worst.setdefault(k, dict(maxrel=0.0, per=0.0, res=0.0, near=e['near_boundary']))
        for key in ('maxrel', 'per', 'res'):
            w[key] = max(w[key], e[key])
    p90 = float(np.percentile(per, 90))
    print(f'\n{label}: {len(dev)} envs, per-contact p90 {p90:.2e}')
    print(f'  {"state":<14} {"nefc":>4} {"cols":>4} {"t/b/m":>8} {"maxrel":>9} {"contact":>9} {"ulps":>6}  near boundary')
    for k, w in sorted(worst.items()):
        p = ss.STATES[NAMES[k]][1]
        print(f'  {NAMES[k]:<14} {p["nefc"]:>4} {p["cols"]:>4} {p["top"]:>2}/{p["bottom"]}/{p["middle"]:<3} {w["maxrel"]:9.2e} {w["per"]:9.2e} '
              f'{w["res"]:6.1f}  {w["near"]}')
    assert not bad, (label, bad[:5])
    assert p90 < PER_P90, (label, p90)
    return p90


def test_analytic_model_keeps_only_closed_form_pairs():
    full = load_model('walk')
    m = model()
    generic = np.isin(full.geom_type, [4, 5])
    assert 0 < m.npair < full.npair and m.c.npair == m.npair == len(m.pair_geom1)
    assert not generic[m.pair_geom1].any() and not generic[m.pair_geom2].any()
    assert m.npair + int((generic[full.pair_geom1] | generic[full.pair_geom2]).sum()) == full.npair
    assert full.npair == len(full.pair_geom1)                   # the copy left the walk model alone


def test_targeted_states_keep_their_properties():
    """each pinned state still reaches its edge at the oracle's Newton optimum (noslip off: the solver's own answer)"""
    m = model(noslip=0)
    for name, (t, want) in ss.STATES.items():
        got = ss.describe(ss.oracle_solution(m, *t), m.opt_impratio)
        assert got == want, (name, t, got, want)
    # with noslip on (the walk model's 3 iterations) the row counts are those of the Newton solve
    for (o, _), name in zip(oracle(), NAMES):
        assert o['nefc'] == ss.STATES[name][1]['nefc'], name


@pytest.fixture(scope='module')
def emu():
    ge.build()
    return ge.EMU


@pytest.fixture(scope='module')
def emu_chol(tmp_path_factory):
    """the host-emulation build with FB_CHOL_REG = 0 (every Hessian block factorised in the record) and 8 (both forms)"""
    return ss.build_chol_variants(tmp_path_factory.mktemp('emu_chol'), ge.CSRC)


@pytest.mark.parametrize('placement', ['default', 'ncap0', 'chol_reg0', 'chol_reg8'])
def test_solver_gates_under_emulation(emu, emu_chol, placement, monkeypatch):
    """the kernel source on the host: all states as envs of one batch, through the register path (default), the generic path for every
    nefc (FB_SOLVE_NCAP = 0) and the record-side Hessian factorisation above 0 / 8 columns"""
    lib = emu
    if placement == 'ncap0':
        monkeypatch.setenv('FB_SOLVE_NCAP', '0')
    elif placement.startswith('chol_reg'):
        lib = emu_chol[int(placement[-1])]
    m = model()
    gate(f'emulation {placement}', st.BatchedStepper(m, len(NAMES), lib_path=lib), m)


def _noslip_effect():
    """largest change of a friction force between noslip 0 and 10 (oracle), relative to the state's largest force"""
    worst = 0.0
    for (a, _), (b, _) in zip(oracle(0), oracle(10)):
        fmax = np.abs(a['force']).max() if a['nefc'] else 1.0
        for adr, dim, _ in ss.contact_rows(a):
            if dim == 3:
                worst = max(worst, float(np.abs(a['force'][adr + 1:adr + 3] - b['force'][adr + 1:adr + 3]).max() / fmax))
    return worst


@pytest.mark.parametrize('noslip', [0, 10])
def test_noslip_settings_under_emulation(emu, noslip):
    """noslip must move friction forces by far more than the gate (else comparing with it on and off proves nothing), and the
    stepper must follow the oracle with it off and with 10 sweeps"""
    effect = _noslip_effect()
    print(f'\nnoslip 0 -> 10 moves a friction force by {effect:.2e} of the largest force')
    assert effect > 20 * MAXREL
    m = model(noslip)
    gate(f'emulation noslip {noslip}', st.BatchedStepper(m, len(NAMES), lib_path=emu), m, noslip=noslip)


def warm_start_errors(m, sim, n_steps, n_sub=10, seed=0, ctrl_scale=0.5):
    """teacher-forced control steps (every control step restarts the stepper from the oracle's state, with the oracle's warm start for
    the first substep's acceleration); the later substeps warm-start the solve from the previous substep's forces matched by row key.
    Per control step: max |dq|, max |dv|, the sensor-mean error and the per-contact efc_force error after the last substep"""
    o = fo.Oracle(m, tolerance=1e-12)
    q0 = reset_qpos(m)
    o.reset(q0)
    sim.reset(q0)
    rs = np.random.RandomState(seed)
    eq, ev, es, ef, skipped = [], [], [], [], 0
    for k in range(n_steps):
        sim.set(st.QPOS, o.qpos)
        sim.set(st.QVEL, o.qvel)
        if m.na:
            sim.set(st.ACT, o.get(fo.ACT))
        sim.set(st.QACC_WARMSTART, o.get(fo.QACC_WARMSTART))
        sim.forward()
        ctrl = rs.uniform(-ctrl_scale, ctrl_scale, m.nu)
        sim.set_control(ctrl)
        o.set(fo.CTRL, ctrl)
        sm_o = o.control_step(n_sub)
        sim.step(n_sub)
        eq.append(np.abs(sim.get(st.QPOS)[0] - o.qpos).max())
        ev.append(np.abs(sim.get(st.QVEL)[0] - o.qvel).max())
        es.append(sensor_mean_error(m, sim.get(st.SENSOR_MEAN)[0], sm_o))
        ne, nc = int(o.get(fo.NEFC)[0]), int(o.get(fo.NCON)[0])
        if int(sim.get(st.NEFC)[0, 0]) != ne or int(sim.get(st.NCON)[0, 0]) != nc:
            skipped += 1                          # a contact or limit switched within the step on one side only
            continue
        ora = dict(nefc=ne, force=o.get(fo.EFC_FORCE), con=o.get(fo.CONTACT).reshape(-1, 16)[:nc])
        dev = dict(nefc=ne, force=np.asarray(sim.get(st.EFC_FORCE)[0][:ne], np.float64),
                   con=np.asarray(sim.get(st.CONTACT)[0], np.float64).reshape(-1, 16)[:nc])
        ef.append(ss.errors(dev, ora, m.opt_impratio)['per'])
    r = dict(p90_q=float(np.percentile(eq, 90)), p90_v=float(np.percentile(ev, 90)), p90_s=float(np.percentile(es, 90)),
             p90_f=float(np.percentile(ef, 90)), max_f=float(np.max(ef)), skipped=skipped, steps=n_steps)
    print('\nwarm start across substeps (analytic walk):', r)
    return r


def test_warm_start_across_substeps_under_emulation(emu):
    m = model()
    r = warm_start_errors(m, st.BatchedStepper(m, 1, lib_path=emu), n_steps=8)
    # measured: p90 |dq| 2.4e-7, |dv| 1.5e-4, sensor mean 2.1e-5, per-contact efc_force 3.3e-4; no step skipped
    assert r['p90_q'] < 6e-7 and r['p90_v'] < 3.7e-4 and r['p90_s'] < 5.4e-5, r
    assert r['p90_f'] < 8.3e-4 and r['skipped'] == 0, r


# ---------------------------------------------------------------------------------------------------------------- on the H100

@pytest.mark.gpu
@pytest.mark.parametrize('placement', ['blob1', 'blob0', 'ncap0'])
def test_solver_gates_on_gpu(placement, monkeypatch):
    """all states as envs of one batch (register-path and generic-path warps share CTAs) with the sweep program in shared memory
    (FB_BLOB = 1), read in place (FB_BLOB = 0), and the generic path for every nefc (FB_SOLVE_NCAP = 0)"""
    if placement == 'ncap0':
        monkeypatch.setenv('FB_SOLVE_NCAP', '0')
    else:
        monkeypatch.setenv('FB_BLOB', placement[-1])
    m = model()
    gate(f'H100 {placement}', st.BatchedStepper(m, len(NAMES)), m)


@pytest.mark.gpu
def test_solver_gates_on_gpu_4096_envs():
    """the configuration bench.py times: 4096 envs, sweep program read in place (the default above 1024 envs).  Env i holds state
    (i + i // 4) mod 14, so every state runs at every warp position of a 4-warp CTA (i mod 4) many times over."""
    m = model()
    n = 4096
    assign = [(i + i // 4) % len(NAMES) for i in range(n)]
    pos = {(a, i % 4) for i, a in enumerate(assign)}
    assert len(pos) == 4 * len(NAMES)
    gate('H100 4096 envs', st.BatchedStepper(m, n), m, assign=assign)


@pytest.mark.gpu
@pytest.mark.parametrize('noslip', [0, 10])
def test_noslip_settings_on_gpu(noslip):
    assert _noslip_effect() > 20 * MAXREL
    m = model(noslip)
    gate(f'H100 noslip {noslip}', st.BatchedStepper(m, len(NAMES)), m, noslip=noslip)


@pytest.mark.gpu
def test_warm_start_across_substeps_on_gpu():
    m = model()
    r = warm_start_errors(m, st.BatchedStepper(m, 32), n_steps=50)
    # measured on an H100: p90 |dq| 2.1e-7, |dv| 2.9e-4, sensor mean 3.0e-5, per-contact efc_force 7.9e-4; no step skipped
    assert r['p90_q'] < 5.3e-7 and r['p90_v'] < 7.3e-4 and r['p90_s'] < 7.5e-5, r
    assert r['p90_f'] < 2e-3 and r['skipped'] <= 2, r
