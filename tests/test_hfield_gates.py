"""The heightfield stage against the fp64 oracle, prism by prism and contact by contact: sphere, capsule, ellipsoid and cylinder on the
pinned cases of tests/hfield_cases.py, first function by function under emulation (fb_emu_convex_hfield_prisms against
orc_convex_hfield_prisms, contacts identified by the triangle they came from), then through the ABI on the fp32-rounded `vision` model
(emulation and H100: the only way to hold the CUDA-compiled prism walk, the bounding-sphere pre-test and the staging), with the
capacities (4 contacts per geom, 64 per env, 125 ... 192 listed geoms) and a bitwise comparison across batch layouts, launch paths
(a permuted batch, each env alone, fb_state_load of a subset) and the two ways a terrain arrives (the device vision task's bank reset,
fb_hfield_write), and finally the full `vision` model dipped into bumps and a trench.

Gates (inputs rounded to fp32 before either side sees them; one unit = 2^-24 of the geom's bounding radius for dist, of max(rbound,
|geom - terrain origin|) for pos -- the device adds the geom's offset back in fp32 -- and 2^-24 for the unit frame vectors; every
heightfield contact comes out of MPR; each stage has its own tolerances, 2.5 x its measurements):
  contact decision (per prism / per pair)    equal, except where a dist of that prism / pair is within MPR_BAND of the margin: reported
  include decision (dist < margin - gap)     equal, except within MPR_BAND of margin - gap
  dist, pos, frame, per function             error <= MPR_K x (the larger of both sides' own spread over fp32-sized perturbations of the
                                             geom's pose) + FIXED_FN; a case where either side jumps under its perturbations (its prisms
                                             change, or an answer moves by more than JUMP) is an MPR discontinuity: reported, counted,
                                             at most JUMPS_FN
  dist, pos, frame, through the ABI          error <= FIXED_ABI / FIXED_FULL; a contact off by more than JUMP is a discontinuity:
                                             reported, counted, at most JUMPS_ABI (none on the full model or at the capacities)
  the 4-per-geom cap                         the kept prisms are the oracle's first ones in walk order, unless an earlier prism's
                                             decision was in band
  pre-test soundness (through the ABI)       every oracle contact below margin - MPR_BAND is on the device
"""
import ctypes as C

import numpy as np
import pytest

import __graft_entry__ as ge
import hfield_cases as hc
from collision_cases import f32, rot_axis, rand_rot
from flybody_b200 import stepper as st
from flybody_b200.flymodel import load_model
from oracle import fly_oracle as fo
from solver_states import fp32_model
from test_collision_gates import quat_of, mat_of

ULP = 2.0 ** -24
# measured under emulation (the kernel source on the host) and on an H100 (80 GB HBM3, 700 W); tolerance = the larger x 2.5
MPR_BAND = 2e-6           # MPR decides contact or none to its tolerance (1e-6): decision flips this close to the margin are reported
MPR_K = 4.0               # per function the device may move as far as 4 x the larger of both sides' own fp32 sensitivity ...
JUMP = 1e6                # an answer that moves by more than this under fp32 perturbations is discontinuous there
# ... plus FIXED_FN units (dist / pos / frame), sized on the cases where neither side jumps.  Worst error - 4 x spread, emulation:
# 1.99e3 (ellipsoid), 0 (a floor of 64), 4.28e5 (ellipsoid); MPR discontinuities (cases where a side's prisms change or an answer moves
# by more than JUMP under its own perturbations): emulation 17 of 625 cases
FIXED_FN, JUMPS_FN = (5.0e3, 64.0, 1.07e6), 42
# through the ABI and on the full model the pose is the kinematics' own, so no spread: a contact off by more than JUMP units is counted
# as a discontinuity, the others are gated on a fixed term.  Worst errors of the others (dist / pos / frame), emulation 2.42e5 / 106 /
# 8.88e5, H100 (80 GB HBM3, 700 W) 1.05e5 / 23.8 / 8.89e5; x 2.5 puts the frame term past JUMP, which then bounds it.  Discontinuities
# in 1385 contacts: emulation 7, H100 11 (capsules and cylinders; the capacity cases: none)
FIXED_ABI, JUMPS_ABI, JUMPS_CAP = (6.05e5, 265.0, JUMP), 28, 0
FIXED_FULL = (1.7e4, 66.0, 1.0e5)         # full model: emulation 6.6e3 / 18.3 / 4.0e4, H100 6.6e3 / 26.2 / 2.6e4
FB_HF_PER_GEOM, FB_MAXCON, FB_MAXCAND = 4, 64, 192


def new_stats():
    return dict(cases=0, contacts=0, band=[], bad=[], jumps=[], worst=np.zeros(3), excess=np.zeros(3))


def table(title, per_type, fixed, max_jumps):
    print(f'\n{title}')
    print(f'  {"geom":<10} {"cases":>5} {"contacts":>8} {"in band":>7} {"outside":>7} {"jumps":>5} {"dist":>9} {"pos":>9} {"normal":>9}'
          f'   worst error, units of 2^-24;  worst error - {MPR_K:g} x spread:')
    for t, s in per_type.items():
        name = hc.NAMES.get(t, t)
        print(f'  {name:<10} {s["cases"]:>5} {s["contacts"]:>8} {len(s["band"]):>7} {len(s["bad"]):>7} {len(s["jumps"]):>5} '
              f'{s["worst"][0]:9.3g} {s["worst"][1]:9.3g} {s["worst"][2]:9.3g}   {s["excess"][0]:9.3g} {s["excess"][1]:9.3g} {s["excess"][2]:9.3g}')
    print(f'  tolerance: {fixed} units (per function: + {MPR_K:g} x spread); MPR discontinuities at most {max_jumps}')
    for t, s in per_type.items():
        for j in s['jumps']:
            print(f'  MPR discontinuity {hc.NAMES.get(t, t)} {j}')
        if s['band']:
            print(f'  inside the band {hc.NAMES.get(t, t)}: {s["band"][:10]}')
    bad = [(hc.NAMES.get(t, t), b) for t, s in per_type.items() for b in s['bad']]
    assert not bad, bad[:8]
    assert sum(len(s['jumps']) for s in per_type.values()) <= max_jumps


def incl(dist, margin, gap):
    return bool(np.float32(dist) < np.float32(np.float32(margin) - np.float32(gap)))


def errors(c, dev, ora):
    """(dist, pos, normal) error of matched contacts [n, 7], in units"""
    if not len(ora):
        return np.zeros(3)
    d = np.abs(dev - ora)
    return np.array([d[:, 0].max() / (ULP * c.rb), d[:, 1:4].max() / (ULP * c.pos_scale), d[:, 4:7].max() / ULP])


def spread(c, ora, opr, rs, run=None, k=4):
    """one side's own spread over k fp32-sized perturbations of the geom's pose, prism by prism (run(p, R) -> (contacts, prism ids);
    default the oracle, moved by 4 units of its position scale and 4 x 2^-24 rad); None where its prisms change (other than in the
    band) or an answer jumps"""
    sp = np.zeros(3)
    omap = dict(zip(opr.tolist(), ora))
    for _ in range(k):
        if run is None:
            o, pr = c.oracle(p=c.p + rs.normal(size=3) * 4 * ULP * c.pos_scale, R=rot_axis(rs.normal(size=3), 4 * ULP) @ c.R)
        else:
            # the device sees fp32 inputs: each coordinate moves by a few of its own fp32 steps, the rotation by 8 x 2^-24 rad
            step = np.maximum(np.spacing(np.abs(c.p).astype(np.float32)).astype(np.float64), 4 * ULP * c.pos_scale)
            o, pr = run(c.p + np.round(rs.normal(size=3) * 4) * step, rot_axis(rs.normal(size=3), 8 * ULP) @ c.R)
        m = dict(zip(pr.tolist(), o))
        for key in set(m) ^ set(omap):
            d = (m.get(key) if key in m else omap[key])[0]
            if abs(d - c.margin) >= MPR_BAND:
                return None
        common = sorted(set(m) & set(omap))
        if common:
            sp = np.maximum(sp, errors(c, np.array([m[q] for q in common]), np.array([omap[q] for q in common])))
    return None if sp.max() > JUMP else sp


def judge(c, dev, dpr, ora, opr, rs, s, run_dev):
    """gate one case, prism by prism (dev, ora [n, 7]; dpr, opr the prism ids; run_dev(p, R): the device on a moved geom).  A case
    where either side jumps under its own fp32-sized perturbations (its prisms change, or an answer moves by more than JUMP units) is an
    MPR discontinuity: reported and counted, its values not gated"""
    s['cases'] += 1
    dmap, omap = dict(zip(dpr.tolist(), dev)), dict(zip(opr.tolist(), ora))
    for key in set(dmap) ^ set(omap):
        d = (dmap[key] if key in dmap else omap[key])[0]
        if abs(d - c.margin) < MPR_BAND:
            s['band'].append(c.name)
        else:
            s['bad'].append((c.name, 'decision', key, 'device' if key in dmap else 'oracle', d))
    common = sorted(set(dmap) & set(omap))
    if not common:
        return
    dv, ov = np.array([dmap[q] for q in common]), np.array([omap[q] for q in common])
    s['contacts'] += len(common)
    for a, b in zip(dv[:, 0], ov[:, 0]):
        if abs(b - (c.margin - c.gap)) < MPR_BAND:
            s['band'].append(c.name)
        elif incl(a, c.margin, c.gap) != incl(b, c.margin, c.gap):
            s['bad'].append((c.name, 'include', a, b))
    e = errors(c, dv, ov)
    so, sd = spread(c, ora, opr, rs), spread(c, dev, dpr, rs, run_dev)
    if so is None or sd is None:
        s['jumps'].append((c.name, 'oracle' if so is None else 'device', e.round(1).tolist()))
        return
    sp = np.maximum(so, sd)
    s['worst'] = np.maximum(s['worst'], e)
    s['excess'] = np.maximum(s['excess'], e - MPR_K * sp)
    if (e > MPR_K * sp + FIXED_FN).any():
        s['bad'].append((c.name, 'mpr', e.tolist(), sp.tolist()))


def judge_cap(c, dpr_cap, dpr, dev, opr_cap, opr, ora, s):
    """the cap keeps the first prisms in walk order: the device's capped list is its own uncapped list cut, and the oracle's unless an
    earlier prism's decision was in band"""
    assert list(dpr_cap) == list(dpr[:len(dpr_cap)]), (c.name, dpr_cap, dpr)
    if list(dpr_cap) == list(opr_cap):
        return
    first = next(i for i in range(max(len(dpr_cap), len(opr_cap))) if i >= min(len(dpr_cap), len(opr_cap)) or dpr_cap[i] != opr_cap[i])
    upto = max([*dpr_cap[:first + 1], *opr_cap[:first + 1]])
    near = [d for q, d in list(zip(dpr, dev[:, 0])) + list(zip(opr, ora[:, 0])) if q <= upto and abs(d - c.margin) < MPR_BAND]
    if near:
        s['band'].append(c.name)
    else:
        s['bad'].append((c.name, 'cap', list(dpr_cap), list(opr_cap)))


# -------------------------------------------------------------------------------------------- a. per function, under emulation

@pytest.fixture(scope='module')
def emu():
    ge.build()
    lib = C.CDLL(ge.EMU)
    lib.fb_emu_convex_hfield_prisms.argtypes = [C.c_int] + [C.c_void_p] * 3 + [C.c_float] + [C.c_void_p] * 3 + [C.c_int, C.c_int] + [C.c_void_p] * 2 + [C.c_int, C.c_void_p]
    return lib


def emu_hf(lib, c, kmax=None):
    kmax = c.kmax if kmax is None else kmax
    f = [np.ascontiguousarray(x, np.float32).ravel() for x in (c.p, c.R, c.s, c.hp, c.hR, c.hsize, c.data)]
    out, pr = np.zeros((kmax, 7), np.float32), np.zeros(kmax, np.int32)
    n = lib.fb_emu_convex_hfield_prisms(c.t, f[0].ctypes.data, f[1].ctypes.data, f[2].ctypes.data, c.margin, f[3].ctypes.data, f[4].ctypes.data,
                                        f[5].ctypes.data, c.data.shape[0], c.data.shape[1], f[6].ctypes.data, out.ctypes.data, kmax, pr.ctypes.data)
    return out[:n].astype(np.float64), pr[:n]


_CASES = {}


def cases():
    if not _CASES:
        _CASES.update(hc.all_cases())
    return _CASES


def test_edge_cases_keep_their_properties():
    for cs in cases().values():
        for c in cs:
            if c.check is not None:
                c.check(c, c.oracle()[0])


def test_hfield_gates_per_function_under_emulation(emu):
    rs = np.random.RandomState(7)
    per_type = {}
    for t, cs in cases().items():
        s = per_type[t] = new_stats()
        for c in cs:
            dev, dpr = emu_hf(emu, c)
            ora, opr = c.oracle()
            judge(c, dev, dpr, ora, opr, rs, s, lambda p, R, c=c: emu_hf(emu, c.moved(c.name, p=p, R=R)))
    counts = {hc.NAMES[t]: sum(len(c.oracle()[0]) > 0 for c in cs) for t, cs in cases().items()}
    print('\ncases with an oracle contact per type:', counts)
    assert min(counts.values()) > 50
    table('heightfield gates, kernel source per function (emulation)', per_type, FIXED_FN, JUMPS_FN)


def test_the_per_geom_cap_keeps_the_first_prisms_in_walk_order(emu):
    rs = np.random.RandomState(9)
    per_type = {}
    for c in hc.cap_cases(hc.terrains()):
        s = per_type.setdefault(c.t, new_stats())
        dev, dpr = emu_hf(emu, c, 50)
        ora, opr = c.oracle(50)
        assert len(opr) >= 6, (c.name, len(opr))
        judge(c, dev, dpr, ora, opr, rs, s, lambda p, R, c=c: emu_hf(emu, c.moved(c.name, p=p, R=R), 50))
        for cap in (FB_HF_PER_GEOM, 50):
            judge_cap(c, emu_hf(emu, c, cap)[1], dpr, dev, c.oracle(cap)[1], opr, ora, s)
    table('heightfield gates, 4-per-geom cap (emulation)', per_type, FIXED_FN, JUMPS_FN)


# ------------------------------------------------------------------------------------ b. the fp32 `vision` model through the ABI

def vision_model(hq=None, hpos=None):
    """the fp32-rounded `vision` model, its terrain geom optionally moved to (hpos, hq)"""
    m = load_model('vision').copy()
    g = m.meta['hf_geom']
    if hq is not None:
        m.a['geom_quat'][g] = hq
    if hpos is not None:
        m.a['geom_pos'][g] = hpos
    return fp32_model(m.rebuild())


def terrain_frame(m):
    g = m.meta['hf_geom']
    return np.asarray(m.geom_pos[g], np.float64), mat_of(np.asarray(m.geom_quat[g], np.float64))


def dipped(m, rs, data, hsize, n, lim=None, dz=(0.0, 0.1), tilt=0.4):
    """qpos [n, nq]: the fly (legs down, wings folded) at random (x, y) of the terrain frame, its thorax dz above the surface there,
    turned by a random yaw and a tilt up to `tilt` rad, all in the terrain's frame"""
    hp, hR = terrain_frame(m)
    lim = 0.99 * hsize[0] - 0.3 if lim is None else lim
    q = np.tile(m.qpos0, (n, 1))
    for i in range(n):
        x, y = rs.uniform(-lim, lim, 2)
        z = hc.height(data, hsize, x, y) + rs.uniform(*dz)
        R = hR @ rot_axis([0, 0, 1], rs.uniform(0, 2 * np.pi)) @ rot_axis(rs.normal(size=3), rs.uniform(0, tilt))
        q[i, 0:3], q[i, 3:7] = hp + hR @ np.array([x, y, z]), quat_of(R)
    return f32(q)


def run(m, q, terr, hsize, pair_geom, lib_path=None, ids=None):
    """forward of qpos rows q with per-env terrains terr [n, nrow, ncol]: (ncon, CONTACT rows [n, 64, 16], FLAGS)"""
    n = len(q)
    sim = st.BatchedStepper(m, n, lib_path=lib_path)
    sim.hfield_collision(m.meta['hf_geom'], hsize, terr.shape[1], terr.shape[2], pair_geom)
    sim.hfield_write(np.arange(n), terr.astype(np.float32))
    sim.reset(q)
    sim.forward()
    out = sim.get(st.NCON)[:, 0].astype(int), np.asarray(sim.get(st.CONTACT)).reshape(n, -1, 16), sim.get(st.FLAGS)[:, 0].astype(int)
    sim.close()
    return out


def oracle_rows(m, q, terr, hsize, pair_geom, count=False):
    """the oracle's first 64 CONTACT rows (and its whole contact count)"""
    o = fo.Oracle(m)
    o.set_hfield(m.meta['hf_geom'], hsize, np.asarray(terr, np.float64), pair_geom)
    o.reset(q)
    o.forward()
    n = int(o.get(fo.NCON)[0])
    rows = np.asarray(o.get(fo.CONTACT), np.float64).reshape(-1, 16)[:n]
    return (rows, n) if count else rows


def by_pair(rows, pair_list):
    """terrain rows [n, 16] split into the listed pairs' runs (each pair's contacts are consecutive, at most FB_HF_PER_GEOM, in pair order;
    no list here holds the same geom twice in a row); the second value says whether every row found its pair"""
    out, i = [], 0
    for g in pair_list:
        k = 0
        while i < len(rows) and int(rows[i, 8]) == int(g) and k < FB_HF_PER_GEOM:
            i, k = i + 1, k + 1
        out.append(rows[i - k:i])
    return out, i == len(rows)


def gate_rows(m, name, drow, orow, pair_list, per_type, fixed, flags=0, maxcon=FB_MAXCON):
    """every CONTACT row of one env against the oracle's: the collision stage's rows with the same geom pairs, then the terrain rows pair
    by pair in walk order.  A pair whose count differs is reported when one of its own contacts (either side) lies within MPR_BAND of the
    margin, else it fails (pre-test soundness: every oracle contact below margin - MPR_BAND is on the device).  Each terrain contact's
    dist, pos and frame (normal and first tangent, CONTACT columns 4:7 and 13:16) within `fixed` units; a contact off by more than JUMP
    units is an MPR discontinuity (the pose is not known here to ask either side for its spread): reported and counted.  The include
    column and the efc addresses are compared where the rows line up and the device's constraint rows did not overflow (FLAGS bit 4:
    it drops the contacts past its row capacity, the oracle does not).  The oracle keeps 256 contacts, the device the first 64."""
    hg = m.meta['hf_geom']
    hp, _ = terrain_frame(m)
    orow, drow = orow[:maxcon], np.asarray(drow, np.float64)
    s = per_type.setdefault('rows', new_stats())
    s['cases'] += 1
    on, dn = orow[orow[:, 7] != hg], drow[drow[:, 7] != hg]
    if not np.array_equal(on[:, 7:9], dn[:, 7:9]):
        s['bad'].append((name, 'collision-stage rows', dn[:, 7:9].tolist(), on[:, 7:9].tolist()))
        return
    (op, ook), (dp_, dok) = by_pair(orow[orow[:, 7] == hg], pair_list), by_pair(drow[drow[:, 7] == hg], pair_list)
    if not (ook and dok):
        s['bad'].append((name, 'terrain rows out of pair order', ook, dok))
        return
    aligned = True
    for k, (a_, b_) in enumerate(zip(dp_, op)):
        shifted = not aligned
        g = int(pair_list[k])
        margin, gap = max(m.geom_margin[hg], m.geom_margin[g]), max(m.geom_gap[hg], m.geom_gap[g])
        if len(a_) != len(b_):
            aligned = False
            if any(abs(r[0] - margin) < MPR_BAND for r in np.r_[a_, b_]):
                s['band'].append(f'{name}/pair{k}')
            elif shifted and len(drow) == maxcon and sum(len(x) for x in dp_[:k + 1]) + len(dn) >= maxcon:
                s['band'].append(f'{name}/pair{k} (cut by the 64-contact cap after an in-band difference)')
            else:
                s['bad'].append((name, f'pair {k} (geom {g}): {len(a_)} device contacts, {len(b_)} oracle', b_[:, 0].tolist()))
            continue
        ts = per_type.setdefault(int(m.geom_type[g]), new_stats())
        rb = float(m.geom_rbound[g])
        for a, b in zip(a_, b_):
            ts['cases'] += 1
            ts['contacts'] += 1
            if not flags & 4 and abs(b[0] - (margin - gap)) >= MPR_BAND and a[10] != b[10]:
                ts['bad'].append((name, 'include', g, a[0], b[0]))
            ps = max(rb, float(np.linalg.norm(b[1:4] - hp)))
            frame = np.r_[4:7, 13:16]
            e = np.array([abs(a[0] - b[0]) / (ULP * rb), np.abs(a[1:4] - b[1:4]).max() / (ULP * ps), np.abs(a[frame] - b[frame]).max() / ULP])
            if (e > JUMP).any():
                ts['jumps'].append((name, g, e.round(1).tolist()))
                continue
            ts['worst'] = np.maximum(ts['worst'], e)
            ts['excess'] = np.maximum(ts['excess'], e)
            if (e > fixed).any():
                ts['bad'].append((name, 'mpr', g, e.round(1).tolist()))
    if aligned and not flags & 4 and not np.array_equal(drow[:, 12], orow[:, 12]):
        s['bad'].append((name, 'efc address', drow[:, 12].tolist(), orow[:, 12].tolist()))


def probe_groups():
    """(name, model, terrains [n, nrow, ncol], hsize, pair list, qpos [n, nq]) per handle"""
    T = hc.terrains()
    base = vision_model()
    pg = np.asarray(base.hf_pair_geom, np.int32)
    hv = f32(base.hf_size)
    bumps, trench = T['bumps'][0], T['trench'][0]
    rs = np.random.RandomState(31)
    out = []
    out.append(('bumps', base, np.stack([bumps] * 27), hv, pg, dipped(base, rs, bumps, hv, 27)))
    out.append(('trench', base, np.stack([trench] * 12), hv, pg, dipped(base, rs, trench, hv, 12)))
    # partly off the terrain: the thorax within 0.3 of the border, outside it
    q = dipped(base, rs, bumps, hv, 8, lim=1.0)
    for i in range(8):
        q[i, i % 2] = (19.85 + 0.05 * (i // 2)) * (1 if i % 4 < 2 else -1)
        q[i, 2] = hc.height(bumps, hv, np.clip(q[i, 0], -20, 20), np.clip(q[i, 1], -20, 20)) + 0.05
    out.append(('border', base, np.stack([bumps] * 8), hv, pg, f32(q)))
    # the window's hmax path: a 401 x 401 grid over a half size of 1 (0.005 cells: most footprints cover more than 64)
    small = f32([1.0, 1.0, 1.0, 0.05])
    fine = f32(0.05 + 0.04 * np.sin(np.linspace(0, 9, 401))[None, :] * np.cos(np.linspace(0, 7, 401))[:, None])
    out.append(('hmax_path', base, np.stack([fine] * 8), small, pg, dipped(base, rs, fine, small, 8, lim=0.7, dz=(0.01, 0.08))))
    # rotated and near-upright terrain frames
    for fname, R, hpos in (('yaw0.012', rot_axis([0, 0, 1], 0.012), [0, 0, -0.01]), ('tilt0.01', rot_axis([1, 0.4, 0], 0.01), [0.1, 0, -0.01]),
                           ('yaw1e-4', rot_axis([0, 0, 1], 1e-4), [0, 0, -0.01]), ('rotated', rand_rot(np.random.RandomState(3)), [0.3, -0.2, 0.5])):
        m = vision_model(quat_of(R), hpos)
        out.append((fname, m, np.stack([bumps] * 12), hv, pg, dipped(m, rs, bumps, hv, 12, dz=(0.02, 0.12))))
    return out


def abi_gates(title, lib_path=None):
    per_type = {}
    for name, m, terr, hs, pg, q in probe_groups():
        ncon, rows, flags = run(m, q, terr, hs, pg, lib_path)
        nt = 0
        for i in range(len(q)):
            orow = oracle_rows(m, q[i], terr[i], hs, pg)
            nt += int((orow[:, 7] == m.meta['hf_geom']).sum())
            gate_rows(m, f'{name}/env{i}', rows[i][:ncon[i]], orow, pg, per_type, FIXED_ABI, flags[i])
        print(f'{name}: {len(q)} envs, {nt} oracle terrain contacts')
        assert nt > len(q), (name, nt)
    table(title, per_type, FIXED_ABI, JUMPS_ABI)


def test_hfield_gates_through_the_abi_under_emulation():
    ge.build()
    abi_gates('heightfield gates, fp32 vision model through the ABI (emulation)', lib_path=ge.EMU)


@pytest.mark.gpu
def test_hfield_gates_through_the_abi_on_gpu():
    abi_gates('heightfield gates, fp32 vision model through the ABI (H100)')


# ------------------------------------------------------------------------------------------------------------- capacities

def capacity_gates(title, lib_path=None):
    """4 contacts per geom, 64 per env (the overflow flag, the oracle's first 64 kept in order) and pair lists of 125 ... 192 geoms
    (the vision model's 70 repeated: every copy of a geom has its contacts, each pair in its own staging slots)"""
    m = vision_model()
    hv = f32(m.hf_size)
    bumps = hc.terrains()['bumps'][0]
    pg = np.asarray(m.hf_pair_geom, np.int32)
    hp, _ = terrain_frame(m)
    x, y = -5.0, 0.0
    q = m.qpos0.copy()
    q[0:3] = [x, y, hc.height(bumps, hv, x, y) - 0.01 + 0.13]     # the pose of the step's terrain parity check
    q = f32(q)
    per_type = {}
    for npair in (70, 125, 126, 140, 192):
        lst = np.resize(pg, npair).astype(np.int32)
        ncon, rows, flags = run(m, q[None], bumps[None], hv, lst, lib_path)
        orow, n_o = oracle_rows(m, q, bumps, hv, lst, count=True)
        over = n_o > FB_MAXCON
        print(f'{title} npair {npair}: oracle {len(orow)} contacts, device {ncon[0]}, FLAGS {flags[0]}')
        assert bool(flags[0] & 2) == over, (npair, flags[0], len(orow))
        gate_rows(m, f'npair{npair}', rows[0][:ncon[0]], orow, lst, per_type, FIXED_ABI, flags[0])
    # more than 64 contacts: the fly pressed into the terrain on its side
    q2 = q.copy()
    q2[2] -= 0.1
    q2[3:7] = quat_of(rot_axis([1, 0, 0], np.pi / 2))
    lst = np.resize(pg, 140).astype(np.int32)
    ncon, rows, flags = run(m, f32(q2)[None], bumps[None], hv, lst, lib_path)
    orow, n_o = oracle_rows(m, f32(q2), bumps, hv, lst, count=True)
    print(f'{title} pressed: oracle {n_o} contacts, device {ncon[0]}, FLAGS {flags[0]}')
    assert n_o > FB_MAXCON and flags[0] & 2 and ncon[0] == FB_MAXCON
    gate_rows(m, 'pressed', rows[0][:ncon[0]], orow, lst, per_type, FIXED_ABI, flags[0])
    table(f'{title}', per_type, FIXED_ABI, JUMPS_CAP)


def test_capacities_under_emulation():
    ge.build()
    capacity_gates('heightfield capacities (emulation)', lib_path=ge.EMU)


@pytest.mark.gpu
def test_capacities_on_gpu():
    capacity_gates('heightfield capacities (H100)')


# ------------------------------------------------------------------------------------------------------- layout invariance

def layout_invariance(lib_path=None):
    """contact rows bitwise equal in a batch of 27 envs (a ragged last block), in a permutation of it, for each env alone, and after
    fb_state_load of a subset (fb_hf_kernel_ids) against the full load"""
    name, m, terr, hs, pg, q = probe_groups()[0]
    n = len(q)
    rs = np.random.RandomState(41)
    terr = np.stack([hc.terrains()['bumps' if i % 2 else 'trench'][0] for i in range(n)])
    q = np.stack([dipped(m, rs, terr[i], hs, 1)[0] for i in range(n)])
    ncon, rows, _ = run(m, q, terr, hs, pg, lib_path)
    assert (ncon > 0).sum() > n // 2
    perm = rs.permutation(n)
    ncon_p, rows_p, _ = run(m, q[perm], terr[perm], hs, pg, lib_path)
    for j, i in enumerate(perm):
        assert ncon_p[j] == ncon[i] and np.array_equal(rows_p[j].view(np.uint32), rows[i].view(np.uint32)), ('permuted', i)
    for i in range(0, n, 3):
        nc1, rows1, _ = run(m, q[i:i + 1], terr[i:i + 1], hs, pg, lib_path)
        assert nc1[0] == ncon[i] and np.array_equal(rows1[0][:ncon[i]].view(np.uint32), rows[i][:ncon[i]].view(np.uint32)), ('alone', i)
    sim = st.BatchedStepper(m, n, lib_path=lib_path)
    sim.hfield_collision(m.meta['hf_geom'], hs, terr.shape[1], terr.shape[2], pg)
    sim.hfield_write(np.arange(n), terr.astype(np.float32))
    sim.reset(q)
    sim.forward()
    sim.state_bank(n)
    sim.save_state()
    far = q.copy()
    far[:, 2] += 3.0
    sim.reset(far)
    sim.forward()
    sub = np.arange(1, n, 2)
    sim.load_state(slots=sub, env_ids=sub)
    nc_s, rows_s = sim.get(st.NCON)[:, 0].astype(int), np.asarray(sim.get(st.CONTACT)).reshape(n, -1, 16)
    sim.load_state()
    nc_f, rows_f = sim.get(st.NCON)[:, 0].astype(int), np.asarray(sim.get(st.CONTACT)).reshape(n, -1, 16)
    sim.close()
    for i in sub:
        assert nc_s[i] == nc_f[i] == ncon[i], ('state load', i, nc_s[i], nc_f[i], ncon[i])
        assert np.array_equal(rows_s[i][:ncon[i]].view(np.uint32), rows_f[i][:ncon[i]].view(np.uint32)), ('subset load', i)
        assert np.array_equal(rows_f[i][:ncon[i]].view(np.uint32), rows[i][:ncon[i]].view(np.uint32)), ('full load', i)


def test_layout_invariance_under_emulation():
    ge.build()
    layout_invariance(ge.EMU)


@pytest.mark.gpu
def test_layout_invariance_on_gpu():
    layout_invariance()


def bank_reset_invariance(lib_path=None):
    """a terrain that arrives through the device vision task's reset (ktask copies the bank's heights, highest point and the eyes'
    block maxima) gives the same contact rows, bit for bit, as the same terrain written with fb_hfield_write.  Every env is first given a flat terrain
    1 below the surface, so a copy that misses the heights or the highest point (the pre-test's bound) changes the rows."""
    from flybody_b200 import fly_envs
    n = 6
    env = fly_envs.vision_guided_flight(n_envs=n, lib_path=lib_path, seed=1, terrain_bank=2, device_task=True)
    sim, m = env._sim, env.model
    bank = np.stack([t for t, _ in env._bank])
    assert not np.array_equal(bank[0], bank[1])
    ids = np.arange(n)
    pick = ids % 2
    sim.hfield_write(ids, np.full((n,) + bank.shape[1:], -1.0, np.float32))
    draws = np.full((n, 8), 0.5, np.float32)
    draws[:, 5] = (pick + 0.5) / 2                    # the terrain draw: bank entry `pick`
    env._forced_draws = draws
    env.reset()
    hv = f32(m.hf_size)
    rs = np.random.RandomState(43)
    q = np.stack([dipped(m, rs, bank[pick[i]].astype(np.float64), hv, 1, lim=15.0)[0] for i in range(n)])
    sim.reset(q)
    sim.forward()
    nc_a, rows_a = sim.get(st.NCON)[:, 0].astype(int), np.asarray(sim.get(st.CONTACT)).reshape(n, -1, 16).copy()
    sim.hfield_write(ids, bank[pick])
    sim.reset(q)
    sim.forward()
    nc_b, rows_b = sim.get(st.NCON)[:, 0].astype(int), np.asarray(sim.get(st.CONTACT)).reshape(n, -1, 16)
    env.close()
    hg = m.meta['hf_geom']
    terrain = [int((rows_b[i][:nc_b[i], 7] == hg).sum()) for i in range(n)]
    print(f'bank reset against fb_hfield_write: terrain contacts per env {terrain}')
    assert sum(t > 0 for t in terrain) >= n // 2, terrain
    for i in range(n):
        assert nc_a[i] == nc_b[i] and np.array_equal(rows_a[i][:nc_a[i]].view(np.uint32), rows_b[i][:nc_b[i]].view(np.uint32)), ('bank', i)


def test_bank_reset_terrain_under_emulation():
    ge.build()
    bank_reset_invariance(ge.EMU)


@pytest.mark.gpu
def test_bank_reset_terrain_on_gpu():
    bank_reset_invariance()


# ------------------------------------------------------------------------------------------------------ c. the full model

VISION_STATES = [('bumps', -5.0, 0.0, 0.13), ('bumps', -5.0, 0.0, 0.17), ('bumps', 3.0, -2.0, 0.11), ('trench', 1.0, 0.5, 0.12),
                 ('trench', -8.0, 3.0, 0.15), ('bumps', 12.0, -7.0, 0.14)]


def full_model_gates(title, lib_path=None):
    """the `vision` model (fp32-rounded) dipped into bumps and a trench at cruising pose, legs down, moving at the parity tests' speed
    (20 along x, random controls): every terrain contact row of the forward pass against the oracle"""
    from flybody_b200 import arenas
    m = fp32_model(load_model('vision'))
    hv = f32(m.hf_size)
    pg = np.asarray(m.hf_pair_geom, np.int32)
    T = hc.terrains()
    rs = np.random.RandomState(0)
    per_type = {}
    nt = 0
    for k, (tn, x, y, dz) in enumerate(VISION_STATES):
        terr = T[tn][0]
        ground = float(arenas.hfield_height(terr.astype(np.float32), [x], [y], 20.0)[0]) - 0.01
        q = m.qpos0.copy()
        q[:3] = [x, y, ground + dz]
        q = f32(q)
        v = np.zeros(m.nv)
        v[0] = 20.0
        ctrl = f32(rs.uniform(-0.2, 0.2, m.nu))
        sim = st.BatchedStepper(m, 1, lib_path=lib_path)
        sim.hfield_collision(m.meta['hf_geom'], hv, 401, 401, pg)
        sim.hfield_write(np.arange(1), terr[None].astype(np.float32))
        sim.reset(q[None], f32(v)[None])
        sim.set_control(ctrl[None].astype(np.float32))
        sim.forward()
        o = fo.Oracle(m)
        o.set_hfield(m.meta['hf_geom'], hv, terr, pg)
        o.reset(q, f32(v))
        o.set(fo.CTRL, ctrl)
        o.forward()
        orow = np.asarray(o.get(fo.CONTACT), np.float64).reshape(-1, 16)[:int(o.get(fo.NCON)[0])]
        nt += int((orow[:, 7] == m.meta['hf_geom']).sum())
        gate_rows(m, f'{tn}{k}', sim.get(st.CONTACT)[0].reshape(-1, 16)[:int(sim.get(st.NCON)[0, 0])], orow, pg, per_type, FIXED_FULL, int(sim.get(st.FLAGS)[0, 0]))
        sim.close()
    print(f'{title}: {nt} oracle terrain contacts')
    assert nt > 20
    table(title, per_type, FIXED_FULL, 0)


def test_full_vision_model_under_emulation():
    ge.build()
    full_model_gates('heightfield gates, full vision model (emulation)', lib_path=ge.EMU)


@pytest.mark.gpu
def test_full_vision_model_on_gpu():
    full_model_gates('heightfield gates, full vision model (H100)')
