"""Constraint-solve states for tests/test_solver_gates.py: the analytic-contact walk model, the pinned table of states that reach
the solver's edges, and the per-contact fp64 gates.

The full walk model has generic convex pairs (ellipsoid / cylinder geoms) whose contact normal and point come from MPR on the device
and from a different narrowphase in the oracle (DESIGN.md section 2): there both sides solve with different J rows, and a solver check
cannot be tighter than the 1e-3 of tests/parity_common.py.  `analytic_model` keeps only the pairs with closed-form contacts (plane,
sphere, capsule), so the oracle and the stepper solve the same problem up to the fp32 rounding of the model, and the solver's own
error can be held about ten times tighter, per contact.
"""
import os
import subprocess

import numpy as np

from flybody_b200 import stepper as st
from flybody_b200.compiler.compile_model import GEOM_CYLINDER, GEOM_ELLIPSOID
from oracle import fly_oracle as fo
from parity_common import random_state

FB_CHOL_REG = 24            # fb_solver_reg.h: Hessian blocks up to this many columns are factorised in registers
FB_SOLVE_NCAP = 32          # fb_solver.h: envs with at most this many rows take the register path

TOP, BOTTOM, MIDDLE = 0, 1, 2          # cone zones of an elliptic contact at the solution: no force, inside the cone, on its surface
ZONE_EPS = 1e-3                        # zone classification slack (relative)
ZONE_BAND = 1e-2                       # a contact this close (relative) to a zone boundary is reported, not gated on its zone
CONE_SLACK = 1e-5                      # fp32 cone feasibility: |f_t / mu| <= f_n (1 + CONE_SLACK)
FLOOR = 1e-4                           # per-contact / per-row error floor, relative to the largest force of the state

# The targeted states: (seed, pos_scale, vel_scale) of parity_common.random_state on analytic_model(walk), found once by a search
# with the oracle, and what the oracle's Newton optimum (noslip off) must look like there.  `cols` counts the active Hessian block
# the way reg_head does; top / bottom / middle count the condim-3 contacts per cone zone.  A model change that moves a state off its
# edge fails test_targeted_states_keep_their_properties instead of quietly testing something else.
STATES = {
    'one_contact':   ((65, 0.1, 1.0),   dict(nefc=3, nlimit=0, ncontact=1, cond1=0, cond3=1, top=0, bottom=1, middle=0, cols=3)),
    'one_limit':     ((48, 0.1, 1.0),   dict(nefc=1, nlimit=1, ncontact=0, cond1=0, cond3=0, top=0, bottom=0, middle=0, cols=1)),
    'nefc31_zones':  ((9, 0.05, 1.0),   dict(nefc=31, nlimit=4, ncontact=9, cond1=0, cond3=9, top=4, bottom=2, middle=3, cols=16)),
    'nefc32':        ((55, 0.05, 1.0),  dict(nefc=32, nlimit=2, ncontact=10, cond1=0, cond3=10, top=4, bottom=1, middle=5, cols=15)),
    'nefc33':        ((13, 0.05, 1.0),  dict(nefc=33, nlimit=0, ncontact=11, cond1=0, cond3=11, top=6, bottom=1, middle=4, cols=11)),
    'zones_generic': ((0, 0.05, 1.0),   dict(nefc=35, nlimit=2, ncontact=11, cond1=0, cond3=11, top=7, bottom=1, middle=3, cols=11)),
    'rows64':        ((114, 0.1, 1.0),  dict(nefc=64, nlimit=1, ncontact=21, cond1=0, cond3=21, top=16, bottom=0, middle=5, cols=11)),
    'rows105':       ((1, 0.2, 1.0),    dict(nefc=105, nlimit=15, ncontact=30, cond1=0, cond3=30, top=26, bottom=4, middle=0, cols=25)),
    'reg_cols24':    ((1109, 0.5, 1.0), dict(nefc=32, nlimit=26, ncontact=2, cond1=0, cond3=2, top=0, bottom=0, middle=2, cols=24)),
    'reg_cols25':    ((1088, 0.5, 1.0), dict(nefc=31, nlimit=24, ncontact=3, cond1=1, cond3=2, top=0, bottom=1, middle=1, cols=25)),
    'reg_condim13':  ((239, 0.3, 1.0),  dict(nefc=15, nlimit=11, ncontact=2, cond1=1, cond3=1, top=0, bottom=0, middle=1, cols=10)),
    'condim13':      ((2, 0.5, 1.0),    dict(nefc=82, nlimit=26, ncontact=20, cond1=2, cond3=18, top=15, bottom=1, middle=2, cols=25)),
    'middle_mu1_a':  ((36, 0.3, 1.0),   dict(nefc=97, nlimit=16, ncontact=27, cond1=0, cond3=27, top=21, bottom=1, middle=5, cols=24)),
    'middle_mu1_b':  ((29, 0.3, 1.0),   dict(nefc=99, nlimit=15, ncontact=28, cond1=0, cond3=28, top=24, bottom=2, middle=2, cols=19)),
}


def build_chol_variants(out_dir, csrc):
    """the host-emulation build of the kernel source with FB_CHOL_REG = 0 (every Hessian block factorised in the record) and 8 (both
    forms), compiled in parallel into out_dir: {0: path, 8: path}"""
    out, procs = {}, []
    for reg in (0, 8):
        out[reg] = os.path.join(str(out_dir), f'libfb_emu_chol{reg}.so')
        procs.append(subprocess.Popen(['g++', '-x', 'c++', '-DFB_EMU', f'-DFB_CHOL_REG={reg}', '-O2', '-std=c++17', '-fPIC', '-shared',
                                       '-o', out[reg], os.path.join(csrc, 'flybody_b200.cu'), '-lm']))
    assert all(p.wait() == 0 for p in procs)
    return out


def analytic_model(m, noslip=None):
    """copy of `m` whose collision pairs exclude every pair with an ellipsoid or cylinder geom; noslip: opt_noslip_iterations"""
    a = m.copy()
    generic = np.isin(a.geom_type, [GEOM_ELLIPSOID, GEOM_CYLINDER])
    keep = ~(generic[a.pair_geom1] | generic[a.pair_geom2])
    a.a['pair_geom1'] = np.ascontiguousarray(a.pair_geom1[keep])
    a.a['pair_geom2'] = np.ascontiguousarray(a.pair_geom2[keep])
    a.a['npair'] = a.meta['npair'] = int(keep.sum())
    if noslip is not None:
        a.a['opt_noslip_iterations'] = a.meta['opt_noslip_iterations'] = int(noslip)
    return a.rebuild()


def fp32_model(m):
    """copy of `m` whose floating-point arrays and options are rounded to fp32: what the stepper's model holds"""
    a = m.copy()
    for k, v in list(a.a.items()):
        if isinstance(v, np.ndarray) and v.dtype == np.float64:
            a.a[k] = v.astype(np.float32).astype(np.float64)
        elif isinstance(v, float) and k.startswith(('opt_', 'stat_')):
            a.a[k] = a.meta[k] = float(np.float32(v))
    return a.rebuild()


def state_inputs(m, seed, pos_scale, vel_scale):
    """qpos, qvel, ctrl of tests/parity_common.random_state's state (seed, pos_scale, vel_scale), rounded to fp32 so that both sides
    start from the same numbers"""
    q, v = random_state(m, seed, pos_scale, vel_scale)
    ctrl = np.random.RandomState(seed + 100).uniform(-0.5, 0.5, m.nu)
    return tuple(x.astype(np.float32).astype(np.float64) for x in (q, v, ctrl))


def oracle_solution(m, seed, pos_scale, vel_scale):
    """the oracle's constraint stage of one state: rows, contacts, forces"""
    o = fo.Oracle(m, tolerance=1e-12)
    q, v, ctrl = state_inputs(m, seed, pos_scale, vel_scale)
    o.reset(q, v)
    o.set(fo.CTRL, ctrl)
    o.forward()
    nefc, ncon = int(o.get(fo.NEFC)[0]), int(o.get(fo.NCON)[0])
    con = o.get(fo.CONTACT).reshape(-1, 16)[:ncon] if ncon else np.zeros((0, 16))
    return dict(nefc=nefc, ncon=ncon, force=o.get(fo.EFC_FORCE), con=con, type=o.efc()['type'],
                niter=int(o.get(fo.SOLVER_NITER)[0]), flags=int(o.get(fo.FLAGS)[0]))


def device_solutions(m, sim, states, assign):
    """reset env i of `sim` to states[assign[i]], one forward; per env: nefc, ncon, forces, contacts, flags"""
    n = sim.n_envs
    inputs = [state_inputs(m, *s) for s in states]
    qs, vs, cs = zip(*[inputs[assign[i]] for i in range(n)])
    sim.reset(np.array(qs), np.array(vs))
    sim.set_control(np.array(cs))
    sim.forward()
    nefc, ncon, flags = sim.get(st.NEFC)[:, 0], sim.get(st.NCON)[:, 0], sim.get(st.FLAGS)[:, 0]
    force, con = sim.get(st.EFC_FORCE), sim.get(st.CONTACT)
    out = []
    for i in range(n):
        ne, nc = int(nefc[i]), int(ncon[i])
        out.append(dict(nefc=ne, ncon=nc, force=np.asarray(force[i][:ne], np.float64), flags=int(flags[i]),
                        con=np.asarray(con[i], np.float64).reshape(-1, 16)[:nc]))
    return out


def contact_rows(sol):
    """(adr, dim, friction) of every contact that has rows; friction is the contact's sliding friction (both tangent directions)"""
    out = []
    for c in sol['con']:
        adr, dim = int(c[12]), int(c[9])
        if adr >= 0:
            out.append((adr, 3 if dim >= 3 else 1, float(c[11])))
    return out


def limit_rows(sol):
    first = min([a for a, _, _ in contact_rows(sol)], default=sol['nefc'])
    return list(range(first))


def zones(sol, impratio=1.0):
    """cone zone of every condim-3 contact from its forces, and its distance to the nearest zone boundary (relative)"""
    f = sol['force']
    fmax = np.abs(f).max() if f.size else 0.0
    out = []
    for adr, dim, mu in contact_rows(sol):
        if dim != 3:
            continue
        fric = mu * np.sqrt(impratio)        # CONTACT holds the regularised cone's mu = friction / sqrt(impratio)
        fn, t = f[adr], np.hypot(f[adr + 1] / fric, f[adr + 2] / fric)
        if fn <= ZONE_EPS * fmax:
            out.append((TOP, np.inf))                     # (zero force: how far the contact is from touching is not in the forces)
        elif t >= fn * (1 - ZONE_EPS):
            out.append((MIDDLE, fn / fmax))               # distance to the top zone
        else:
            out.append((BOTTOM, min(1 - t / fn, fn / fmax)))   # to the cone surface, to the top zone
    return out


def hessian_columns(sol, impratio=1.0):
    """columns of the active Hessian block at this solution (fb_solver_reg.h reg_head): 1 per active plain row (limit, condim-1
    contact), 3 per bottom-zone contact, 2 per middle-zone contact"""
    f = sol['force']
    plain = limit_rows(sol) + [a for a, d, _ in contact_rows(sol) if d == 1]
    n = int(sum(f[r] > 0 for r in plain))
    for z, _ in zones(sol, impratio):
        n += {TOP: 0, BOTTOM: 3, MIDDLE: 2}[z]
    return n


def describe(sol, impratio=1.0):
    z = [zz for zz, _ in zones(sol, impratio)]
    dims = [d for _, d, _ in contact_rows(sol)]
    return dict(nefc=sol['nefc'], nlimit=len(limit_rows(sol)), ncontact=len(dims), cond1=dims.count(1), cond3=dims.count(3),
                top=z.count(TOP), bottom=z.count(BOTTOM), middle=z.count(MIDDLE), cols=hessian_columns(sol, impratio))


def errors(dev, ora, impratio=1.0):
    """fp64 gates of one state: (max-relative efc_force error, worst per-contact / per-limit-row error, worst cone violation,
    zone mismatches outside the boundary band, contacts inside the band); dev and ora must have the same rows"""
    fo_, fd = ora['force'], dev['force']
    fmax = np.abs(fo_).max() if fo_.size else 0.0
    maxrel = float(np.abs(fd - fo_).max() / (fmax + 1e-30)) if fo_.size else 0.0
    floor = FLOOR * fmax
    per = [float(abs(fd[r] - fo_[r]) / (abs(fo_[r]) + floor + 1e-30)) for r in limit_rows(ora)]
    for adr, dim, _ in contact_rows(ora):
        per.append(float(np.abs(fd[adr:adr + dim] - fo_[adr:adr + dim]).max() / (abs(fo_[adr]) + floor + 1e-30)))
    cone = 0.0
    for adr, dim, mu in contact_rows(dev):
        if dim == 3:
            fric = mu * np.sqrt(impratio)
            t = np.hypot(fd[adr + 1] / fric, fd[adr + 2] / fric)
            cone = max(cone, float((t - fd[adr]) / (abs(fd[adr]) + 1e-30)) if t > fd[adr] else 0.0)
    zd, zo = zones(dev, impratio), zones(ora, impratio)
    mismatch = [i for i, ((a, _), (b, eps)) in enumerate(zip(zd, zo)) if a != b and eps >= ZONE_BAND]
    near = [i for i, (_, eps) in enumerate(zo) if eps < ZONE_BAND]
    return dict(maxrel=maxrel, per=max(per, default=0.0), per_all=per, cone=cone, zone_mismatch=mismatch, near_boundary=near)


def jar_resolution(m, seed, pos_scale, vel_scale):
    """per row: D_r * (|J_r| |qacc_smooth| + |aref_r| + sum_j |A_rj f_j|) at the oracle's solution -- the size of the terms that
    cancel in jar_r = J_r qacc_smooth - aref_r + (A f)_r, times the row's stiffness.  An fp32 evaluation of jar cannot resolve
    f_r better than about 2^-24 times this: where it is 1e4 times |f_r| (a light contact under heavy limit and contact forces)
    the fp32 solve is 1e-3 - 1e-2 off relative to that contact's own force, whatever the solver does."""
    o = fo.Oracle(m, tolerance=1e-12)
    q, v, ctrl = state_inputs(m, seed, pos_scale, vel_scale)
    o.reset(q, v)
    o.set(fo.CTRL, ctrl)
    o.forward()
    e, nv = o.efc(), m.nv
    M = o.get(fo.QM_DENSE).reshape(nv, nv)
    A = e['J'] @ np.linalg.solve(M, e['J'].T)
    qacc_smooth = np.linalg.solve(M, o.get(fo.QFRC_SMOOTH))
    f = o.get(fo.EFC_FORCE)
    return e['D'] * (np.abs(e['J']) @ np.abs(qacc_smooth) + np.abs(e['aref']) + np.abs(A) @ np.abs(f))
