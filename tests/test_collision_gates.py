"""The collision stage against the fp64 oracle, contact by contact: every pair type of the narrowphase dispatch on the pinned cases of
tests/collision_cases.py, first function by function under emulation (fb_emu_pair against orc_pair), then through the ABI on a probe
model (emulation and H100: the only way to hold the CUDA-compiled narrowphase and MPR per contact), on the full walk and flight
models at the parity tests' random states, on the H100's pooled MPR path (a block's four envs share warp 0's lanes) with chosen job
distributions and a bitwise comparison across batch layouts, and at the candidate (192) and contact (64) capacities.

Gates (inputs rounded to fp32 before either side sees them; one unit = 2^-24 of the pair's scale, the sum of the geoms' bounding radii,
for dist and pos, and 2^-24 for the unit frame vectors; tolerance = measured x 2.5, both measurements beside each constant):
  contact count and the include decision (dist < margin - gap)   equal, except where the oracle's dist is within BAND units of the
                                                                 margin (count) or of margin - gap (include): reported, not gated;
                                                                 through the ABI also the constraint stages' own decision (CONTACT[10])
  analytic pairs: dist, pos, frame                               worst error <= DIST / POS / FRAME units
  MPR pairs: dist, pos, frame                                    error <= MPR_K x (the oracle's own spread over fp32-sized pose
                                                                 perturbations) + MPR_FIXED units; a case where the oracle itself
                                                                 jumps (its count or answer moves by more than JUMP units under the
                                                                 perturbations) is an MPR discontinuity: printed, at most MPR_JUMPS
  prefilter soundness                                            where the kernel has no generic contact, the oracle's dist is above
                                                                 margin - BAND units
"""
import copy

import numpy as np
import pytest

import __graft_entry__ as ge
import collision_cases as cc
from flybody_b200 import stepper as st
from flybody_b200.compiler.compile_model import rbound
from flybody_b200.flymodel import load_model
from oracle import fly_oracle as fo
from parity_common import random_state
from solver_states import fp32_model

ULP = 2.0 ** -24
# measured under emulation (the kernel source on the host) and on an H100 (80 GB HBM3, 700 W); the larger of the two x 2.5
BAND = 64                 # fp32 decision band around the margin and margin - gap (analytic dist carries at most 22 units of rounding)
DIST = 55                 # emulation 3.0 (probe plane-ellipsoid), H100 21.6 (probe plane-cylinder tilted_3)
POS = 28                  # emulation 2.6 (probe plane-ellipsoid), H100 11.3 (probe plane-cylinder tilted_3)
FRAME = 9                 # emulation 3.4 (probe capsule-capsule), H100 3.6 (probe sphere-sphere)
MPR_K = 4.0               # the device may move as far as 4 x the oracle's own fp32 sensitivity ...
MPR_FIXED = 1.3e5         # ... plus this (MPR stops at a 1e-6 tolerance): emulation 5.2e4 (pooled ellipsoid-cylinder frame), H100 2.2e4
                          # (probe sphere-cylinder dist)
MPR_BAND = 2e-6           # MPR decides contact or none to its tolerance (1e-6): count flips this close to the margin are reported
JUMP = 1e6                # an oracle answer that moves by more than this under fp32 perturbations is discontinuous there
MPR_JUMPS = 0             # disagreements where the oracle itself jumps: emulation 0, H100 0
# the full models add the fp32 kinematics of a 7-joint leg chain to every contact: emulation 104 / 92 / 27, H100 97 / 109 / 19
REAL = (260, 275, 70)     # dist, pos, frame (plane-capsule, both)


_CASES = {}


def cases():
    if not _CASES:
        _CASES.update(cc.all_cases())
    return _CASES


def label(pair):
    return f'{cc.NAMES[pair[0]]}-{cc.NAMES[pair[1]]}'


# --------------------------------------------------------------------------------------------------------------- the gates

def incl(dist, margin, gap):
    """the include decision as both sides make it: dist < margin - gap, in fp32 on the device"""
    return bool(np.float32(dist) < np.float32(np.float32(margin) - np.float32(gap)))


def perturbed(c, rs, k):
    """c with both poses moved by fp32-sized amounts (positions by a few units of the scale, rotations by a few 2^-24 rad)"""
    out = []
    for _ in range(k):
        d = {}
        for p, R, t in (('p1', 'R1', c.t1), ('p2', 'R2', c.t2)):
            if t == cc.PLANE:
                continue
            d[p] = getattr(c, p) + rs.normal(size=3) * 4 * ULP * c.scale
            d[R] = cc.rot_axis(rs.normal(size=3), 4 * ULP) @ getattr(c, R)
        q = cc.Case(**{**c.__dict__, **d})
        q.__dict__.update(d)                  # keep the perturbation in fp64
        out.append(q)
    return out


def sensitivity(c, ora, rs, k=4):
    """the oracle's own spread (dist, pos, frame in units) over k perturbations of the pose; None where it jumps"""
    sp = np.zeros(3)
    for q in perturbed(c, rs, k):
        o = q.oracle()
        if len(o) != len(ora):
            return None
        sp = np.maximum(sp, errors(c, o, ora))
    return None if sp.max() > JUMP else sp


def errors(c, dev, ora):
    """worst (dist, pos, frame) error of matched contacts, in units"""
    L = ULP * c.scale
    d = np.abs(dev - ora)
    return np.array([d[:, 0].max() / L, d[:, 1:4].max() / L, d[:, 4:13].max() / ULP]) if len(ora) else np.zeros(3)


def match_order(dev, ora):
    """order of the device contacts that meets each oracle contact with the device contact nearest to it: the contacts of one pair
    that tie (the two ends of a cylinder lying flat) come in an order decided by the sign of a rounded zero"""
    if len(dev) != len(ora):
        return np.arange(len(dev))
    free, order = list(range(len(dev))), []
    for o in ora:
        j = min(free, key=lambda j: np.abs(dev[j, 1:4] - o[1:4]).max())
        free.remove(j)
        order.append(j)
    return np.array(order, int)


def judge(c, dev, ora, rs, stats, dinc=None, oinc=None):
    """gate one case (dev, ora: [n, 13] contacts; dinc, oinc: the include decisions both sides' constraint stages made, where they
    are read through the ABI); stats collects the pair type's row of the table"""
    L = ULP * c.scale
    generic = c.pair not in cc.ANALYTIC
    stats['cases'] += 1
    band = max(BAND * L, MPR_BAND) if generic else BAND * L
    near_margin = any(abs(d - c.margin) < band for d in np.r_[ora[:, 0], dev[:, 0]])
    if len(dev) != len(ora):
        if near_margin:
            stats['band'].append(c.name)
        elif generic and sensitivity(c, ora, rs) is None:
            stats['jumps'].append((c.name, f'count {len(dev)} vs {len(ora)}'))
        else:
            stats['bad'].append((c.name, 'pruned' if generic and len(dev) == 0 else f'count {len(dev)} vs {len(ora)}',
                                 ora[:, 0].tolist(), dev[:, 0].tolist()))
        return
    order = match_order(dev, ora)
    dev = dev[order]
    incl_band = max(BAND * L, MPR_BAND) if generic else BAND * L
    for i, (a, b) in enumerate(zip(dev[:, 0], ora[:, 0])):
        if abs(b - (c.margin - c.gap)) < incl_band:
            stats['band'].append(c.name)
        elif incl(a, c.margin, c.gap) != incl(b, c.margin, c.gap):
            stats['bad'].append((c.name, 'include (dist)', a, b))
        elif dinc is not None and dinc[order[i]] != oinc[i]:
            stats['bad'].append((c.name, 'include (constraint stage)', a, b, dinc[order[i]], oinc[i]))
    e = errors(c, dev, ora)
    if generic:
        sp = sensitivity(c, ora, rs)
        if sp is None and (near_margin or (e <= MPR_FIXED).all()):
            return                            # the oracle jumps here, and the kernel agrees with one of its answers
        if sp is None:
            stats['jumps'].append((c.name, e.round(1).tolist()))
            return
        stats['worst'] = np.maximum(stats['worst'], e)
        stats['spread'] = np.maximum(stats['spread'], sp)
        if (e > MPR_K * sp + MPR_FIXED).any():
            stats['bad'].append((c.name, 'mpr', e.tolist(), sp.tolist()))
    else:
        stats['worst'] = np.maximum(stats['worst'], e)
        if (e > [DIST, POS, FRAME]).any():
            stats['bad'].append((c.name, 'analytic', e.tolist()))


def new_stats():
    return dict(cases=0, band=[], bad=[], jumps=[], worst=np.zeros(3), spread=np.zeros(3))


def table(title, per_pair):
    print(f'\n{title}')
    print(f'  {"pair":<22} {"cases":>5} {"in band":>7} {"outside":>7} {"jumps":>5} {"dist":>9} {"pos":>9} {"frame":>9}   (units of 2^-24)')
    for pair, s in per_pair.items():
        print(f'  {label(pair):<22} {s["cases"]:>5} {len(s["band"]):>7} {len(s["bad"]):>7} {len(s["jumps"]):>5} '
              f'{s["worst"][0]:9.1f} {s["worst"][1]:9.1f} {s["worst"][2]:9.1f}')
    for pair, s in per_pair.items():
        for j in s['jumps']:
            print(f'  MPR discontinuity {label(pair)} {j}')
        if s['band']:
            print(f'  inside the band {label(pair)}: {s["band"]}')
    bad = [(label(p), b) for p, s in per_pair.items() for b in s['bad']]
    jumps = sum(len(s['jumps']) for s in per_pair.values())
    assert not bad, bad[:8]
    assert jumps <= MPR_JUMPS, jumps


# -------------------------------------------------------------------------------------------- a. per function, under emulation

@pytest.fixture(scope='module')
def emu():
    import ctypes as C
    ge.build()
    lib = C.CDLL(ge.EMU)
    lib.fb_emu_pair.argtypes = [C.c_int] + [C.c_void_p] * 3 + [C.c_int] + [C.c_void_p] * 3 + [C.c_float, C.c_void_p]
    return lib


def emu_pair(lib, c):
    f = [np.ascontiguousarray(x, np.float32).ravel() for x in (c.p1, c.R1, c.s1, c.p2, c.R2, c.s2)]
    out = np.zeros((4, 13), np.float32)
    n = lib.fb_emu_pair(c.t1, *[x.ctypes.data for x in f[:3]], c.t2, *[x.ctypes.data for x in f[3:]], c.margin, out.ctypes.data)
    return out[:n].astype(np.float64)


def test_edge_cases_keep_their_properties():
    for pair, cs in cc.edge_cases().items():
        for c in cs:
            c.check(c, c.oracle())


def test_collision_gates_per_function_under_emulation(emu):
    rs = np.random.RandomState(7)
    per_pair = {}
    for pair, cs in cases().items():
        s = per_pair[pair] = new_stats()
        for c in cs:
            judge(c, emu_pair(emu, c), c.oracle(), rs, s)
    table('collision gates, kernel source per function (emulation)', per_pair)


@pytest.mark.parametrize('name', [f'near_parallel_{th:.0e}' for th in (1e-2, 1e-3, 1e-4, 1e-5, 1e-6)] +
                         [f'near_parallel_rotated_{th:.0e}' for th in (1e-6, 1e-7)])
def test_near_parallel_capsules_take_the_oracles_branch(emu, name):
    """two capsules 1e-2 ... 1e-7 rad off parallel (the world frame, and a rotated one): one contact where the fp64 reference has
    one, at its place (the fp32 determinant 1 - cos^2 used to vanish below 2.4e-4 rad and send them to the parallel branch: two
    contacts at other places)"""
    c = {x.name: x for x in cc.edge_cases()[(cc.CAP, cc.CAP)]}[name]
    dev, ora = emu_pair(emu, c), c.oracle()
    assert len(dev) == len(ora) == 1, (dev, ora)
    e = errors(c, dev, ora)
    print(f'\ncapsule-capsule {name}: dist / pos / frame error {e.round(1)} units')
    assert (e < [DIST, POS, FRAME]).all(), e


def test_prefilter_prunes_only_pairs_without_a_contact(emu):
    """DESIGN.md: the generic pairs' prefilter "does not change any result".  On the cases placed within 2e-5 of the margin, wherever
    the kernel source returns no contact the oracle's dist is above the margin less the fp32 band, and each near case is decided"""
    pruned = kept = 0
    for pair, cs in cases().items():
        for c in cs:
            if pair in cc.ANALYTIC or not c.name.startswith('near'):
                continue
            dev, ora = emu_pair(emu, c), c.oracle()
            if len(dev) == 0:
                pruned += 1
                assert all(d > c.margin - BAND * ULP * c.scale for d in ora[:, 0]), (label(pair), c.name, ora[:, 0])
            else:
                kept += 1
    print(f'\nprefilter: {pruned} near cases without a contact, {kept} with one')
    assert pruned > 20 and kept > 20


# --------------------------------------------------------------------------------------------- b. a probe model through the ABI

THORAX = 1


def quat_of(R):
    """unit quaternion (w, x, y, z) of a rotation matrix"""
    w = np.sqrt(max(0.0, 1 + R[0, 0] + R[1, 1] + R[2, 2])) / 2
    x = np.sqrt(max(0.0, 1 + R[0, 0] - R[1, 1] - R[2, 2])) / 2 * np.sign(R[2, 1] - R[1, 2] or 1)
    y = np.sqrt(max(0.0, 1 - R[0, 0] + R[1, 1] - R[2, 2])) / 2 * np.sign(R[0, 2] - R[2, 0] or 1)
    z = np.sqrt(max(0.0, 1 - R[0, 0] - R[1, 1] + R[2, 2])) / 2 * np.sign(R[1, 0] - R[0, 1] or 1)
    q = np.array([w, x, y, z])
    return q / np.linalg.norm(q)


def mat_of(q):
    w, x, y, z = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def probe_model(pair, s1, s2, margin, gap):
    """the walk model with geom 1 on the thorax and the last geom on the ghost body, of the pair's types and sizes at their bodies'
    origins, and one collision pair: those two geoms, or the floor (geom 0) and the ghost geom"""
    m = load_model('walk').copy()
    a = m.a
    ng, ghost = m.ngeom, m.nbody - 1
    g1, g2 = (0 if pair[0] == cc.PLANE else THORAX), ng - 1
    a['geom_bodyid'][THORAX] = THORAX
    a['geom_bodyid'][g2] = ghost
    for g, t, s in ((THORAX, cc.SPH if pair[0] == cc.PLANE else pair[0], s1 if pair[0] != cc.PLANE else [0.01, 0, 0]), (g2, pair[1], s2)):
        a['geom_type'][g] = t
        a['geom_size'][g] = s
        a['geom_pos'][g] = 0
        a['geom_quat'][g] = [1, 0, 0, 0]
        a['geom_rbound'][g] = rbound(t, np.asarray(s))
        a['geom_margin'][g], a['geom_gap'][g] = margin, gap
    a['pair_geom1'] = np.array([g1], np.int32)
    a['pair_geom2'] = np.array([g2], np.int32)
    a['npair'] = m.meta['npair'] = 1
    return fp32_model(m.rebuild())


def probe_qpos(m, cs):
    """per case: the thorax at geom 1's pose (a plane case: at geom 2's, where no pair reaches it) and the ghost at geom 2's,
    rotations as fp32 quaternions; returns qpos [n, nq] and the cases with the rotations both sides' kinematics make of them"""
    gq = m.jnt_qposadr[-1]
    q = np.tile(m.qpos0, (len(cs), 1))
    poses = []
    for i, c in enumerate(cs):
        plane = c.t1 == cc.PLANE
        q1, q2 = cc.f32(quat_of(c.R2 if plane else c.R1)), cc.f32(quat_of(c.R2))
        q[i, 0:3], q[i, 3:7], q[i, gq:gq + 3], q[i, gq + 3:gq + 7] = (c.p2 if plane else c.p1), q1, c.p2, q2
        p = copy.copy(c)
        p.R2 = mat_of(q2)
        if not plane:
            p.R1 = mat_of(q1)
        poses.append(p)
    return cc.f32(q), poses


def contacts(rows, n):
    """[n, 13] contacts (dist, pos, frame) from CONTACT rows: the frame's normal, first tangent and normal x tangent"""
    r = np.asarray(rows, np.float64).reshape(-1, 16)[:n]
    return np.hstack([r[:, 0:7], r[:, 13:16], np.cross(r[:, 4:7], r[:, 13:16])]), r


def probe_gates(title, lib_path=None, per_type=24):
    """every pair type on its probe model, both margin settings: per_type random cases of one size pair, and the type's edge cases"""
    rs = np.random.RandomState(11)
    edges = cc.edge_cases()
    per_pair = {}
    for pair in cc.PAIR_TYPES:
        s = per_pair[pair] = new_stats()
        size_rs = np.random.RandomState(100 + 10 * pair[0] + pair[1])
        s1 = [0, 0, 0] if pair[0] == cc.PLANE else cc.rand_size(pair[0], size_rs)
        s2 = cc.rand_size(pair[1], size_rs)
        for margin, gap in cc.MARGINS:
            cs = cc.random_cases(pair, rs, per_type, sizes=(s1, s2), margins=((margin, gap),))
            by_size = {}
            for e in edges.get(pair, []):
                if (e.margin, e.gap) == (np.float32(margin), np.float32(gap)):
                    by_size.setdefault((tuple(e.s1), tuple(e.s2)), []).append(e)
            for sizes, group in [((tuple(cc.f32(s1)), tuple(cc.f32(s2))), cs)] + list(by_size.items()):
                m = probe_model(pair, *sizes, margin, gap)
                q, poses = probe_qpos(m, group)
                sim = st.BatchedStepper(m, len(group), lib_path=lib_path)
                sim.reset(q)
                sim.forward()
                nc, rows = sim.get(st.NCON)[:, 0], sim.get(st.CONTACT)
                for i, c in enumerate(poses):
                    o = fo.Oracle(m)
                    o.reset(q[i])
                    o.forward()
                    ora, orow = contacts(o.get(fo.CONTACT), int(o.get(fo.NCON)[0]))
                    dev, drow = contacts(rows[i], int(nc[i]))
                    assert np.array_equal(drow[:, 7:9], orow[:, 7:9]) or len(drow) != len(orow), (c.name, drow[:, 7:9], orow[:, 7:9])
                    judge(c, dev, ora, rs, s, drow[:, 10], orow[:, 10])
    table(title, per_pair)


def test_collision_gates_probe_model_under_emulation():
    ge.build()
    probe_gates('collision gates, probe model through the ABI (emulation)', lib_path=ge.EMU)


@pytest.mark.gpu
def test_collision_gates_probe_model_on_gpu():
    probe_gates('collision gates, probe model through the ABI (H100)')


# --------------------------------------------------------------------------------------------------------- e. the real models

STATES = [('walk', 0, 0.05, 1.0), ('walk', 2, 0.05, 1.0), ('walk', 4, 0.0, 1.0), ('walk', 1, 0.2, 1.0), ('flight', 1, 0.05, 20.0)]


def real_model_gates(title, lib_path=None):
    """every contact of the full walk and flight models at the parity tests' random states (one env each), matched by (geom1, geom2,
    ordinal within the pair), against the oracle on the fp32-rounded model"""
    rs = np.random.RandomState(13)
    per_pair = {}
    for variant, seed, ps, vs in STATES:
        m = fp32_model(load_model(variant))
        q, v = random_state(m, seed, ps, vs)
        q = cc.f32(q)
        sim = st.BatchedStepper(m, 1, lib_path=lib_path)
        sim.reset(q[None])
        sim.forward()
        o = fo.Oracle(m)
        o.reset(q)
        o.forward()
        dev, drow = contacts(sim.get(st.CONTACT)[0], int(sim.get(st.NCON)[0, 0]))
        ora, orow = contacts(o.get(fo.CONTACT), int(o.get(fo.NCON)[0]))
        key = lambda r: [(int(a), int(b)) for a, b in r[:, 7:9]]
        dk, ok = key(drow), key(orow)
        assert int(sim.get(st.FLAGS)[0, 0]) & 2 == 0
        for g in sorted(set(dk) | set(ok)):
            di, oi = [i for i, k in enumerate(dk) if k == g], [i for i, k in enumerate(ok) if k == g]
            t1, t2 = int(m.geom_type[g[0]]), int(m.geom_type[g[1]])
            c = cc.Case(f'{variant}{seed}:{g[0]}-{g[1]}', t1, np.zeros(3), cc.EYE, m.geom_size[g[0]], t2, np.zeros(3), cc.EYE,
                        m.geom_size[g[1]], max(m.geom_margin[g[0]], m.geom_margin[g[1]]), max(m.geom_gap[g[0]], m.geom_gap[g[1]]))
            s = per_pair.setdefault((t1, t2), new_stats())
            # the generic pairs' sensitivity is not known here without the oracle's geom poses: gate them on MPR_FIXED alone
            s['cases'] += 1
            band = MPR_BAND if (t1, t2) not in cc.ANALYTIC else BAND * ULP * c.scale
            if len(di) != len(oi):
                if any(abs(d - c.margin) < band for d in np.r_[ora[oi, 0], dev[di, 0]]):
                    s['band'].append(c.name)
                else:
                    s['bad'].append((c.name, 'count', len(di), len(oi)))
                continue
            order = match_order(dev[di], ora[oi])
            for i, k in enumerate(oi):
                if abs(ora[k, 0] - (c.margin - c.gap)) >= band and drow[di[order[i]], 10] != orow[k, 10]:
                    s['bad'].append((c.name, 'include', dev[di[order[i]], 0], ora[k, 0]))
            e = errors(c, dev[di][order], ora[oi])
            s['worst'] = np.maximum(s['worst'], e)
            lim = REAL if (t1, t2) in cc.ANALYTIC else [MPR_FIXED] * 3
            if (e > lim).any():
                s['bad'].append((c.name, e.round(1).tolist()))
    table(title, per_pair)


def test_collision_gates_real_models_under_emulation():
    ge.build()
    real_model_gates('collision gates, walk and flight models (emulation)', lib_path=ge.EMU)


@pytest.mark.gpu
def test_collision_gates_real_models_on_gpu():
    real_model_gates('collision gates, walk and flight models (H100)')


# --------------------------------------------------------------------------- c. the pooled MPR jobs of a block's envs (H100)

GENERIC_K = 6              # generic geoms on each body of the pooled-MPR probe model: 36 generic pairs, all MPR jobs when overlapping
FAR, DEEP = 1.0, 0.004     # ghost-thorax distance of an env without candidates, and of one whose 36 pairs all overlap deeply
FB_WPB = 4                 # envs (warps) per block: the pooled path deals the MPR jobs of these four envs out on warp 0


def multi_model(types1, sizes1, types2, sizes2, pos1=None, quat1=None, pos2=None, quat2=None, margin=0.0, gap=0.0):
    """the walk model with geoms 1..k1 on the thorax and the last k2 geoms on the ghost body (types, sizes, local poses given; default
    at the body's origin) and the collision pairs (thorax geom i, ghost geom j), i-major, lower type first"""
    m = load_model('walk').copy()
    a = m.a
    ng, ghost, k1, k2 = m.ngeom, m.nbody - 1, len(types1), len(types2)
    g1s, g2s = list(range(1, 1 + k1)), list(range(ng - k2, ng))
    for gs, body, types, sizes, pos, quat in ((g1s, THORAX, types1, sizes1, pos1, quat1), (g2s, ghost, types2, sizes2, pos2, quat2)):
        for n, g in enumerate(gs):
            a['geom_bodyid'][g] = body
            a['geom_type'][g] = types[n]
            a['geom_size'][g] = sizes[n]
            a['geom_pos'][g] = 0 if pos is None else pos[n]
            a['geom_quat'][g] = [1, 0, 0, 0] if quat is None else quat[n]
            a['geom_rbound'][g] = rbound(types[n], np.asarray(sizes[n], np.float64))
            a['geom_margin'][g], a['geom_gap'][g] = margin, gap
    assert all(types1[i] <= types2[j] for i in range(k1) for j in range(k2))
    a['pair_geom1'] = np.array([g for g in g1s for _ in g2s], np.int32)
    a['pair_geom2'] = np.array([g for _ in g1s for g in g2s], np.int32)
    a['npair'] = m.meta['npair'] = k1 * k2
    return fp32_model(m.rebuild())


def body_poses(m, q):
    """fp64 world poses (pos, R) of every geom of the thorax and the ghost body at qpos q, as the oracle's kinematics makes them"""
    gq = m.jnt_qposadr[-1]
    out = {}
    for g in range(m.ngeom):
        b = int(m.geom_bodyid[g])
        if b == THORAX:
            bp, bR = q[0:3], mat_of(q[3:7])
        elif b == m.nbody - 1:
            bp, bR = q[gq:gq + 3], mat_of(q[gq + 3:gq + 7])
        else:
            continue
        out[g] = (bp + bR @ m.geom_pos[g], bR @ mat_of(m.geom_quat[g]))
    return out


def pair_case(m, poses, g1, g2):
    (p1, R1), (p2, R2) = poses[g1], poses[g2]
    c = cc.Case(f'{g1}-{g2}', int(m.geom_type[g1]), p1, R1, m.geom_size[g1], int(m.geom_type[g2]), p2, R2, m.geom_size[g2],
                max(m.geom_margin[g1], m.geom_margin[g2]), max(m.geom_gap[g1], m.geom_gap[g2]))
    c.p1, c.R1, c.p2, c.R2 = p1, R1, p2, R2          # the fp64 poses, not rounded again
    return c


def pooled_model():
    ell = lambda r: [r, 1.1 * r, 1.25 * r]
    rs = [0.008 * (i + 1) for i in range(GENERIC_K)]
    t2 = [cc.ELL if i % 2 == 0 else cc.CYL for i in range(GENERIC_K)]
    return multi_model([cc.ELL] * GENERIC_K, [ell(r) for r in rs], t2, [ell(r) if t == cc.ELL else [r, 1.2 * r, 0] for t, r in zip(t2, rs)],
                       margin=5e-4, gap=5e-4)


def pooled_batch(m):
    """27 envs (a ragged last block) whose blocks hold the job distributions the pooled path must handle; per env the ghost's distance
    from the thorax: FAR (no candidate), DEEP (36 jobs) or in between (some)"""
    rs = np.random.RandomState(21)
    mid = lambda: rs.uniform(0.02, 0.1)
    dists = ([FAR, FAR, FAR, DEEP] +            # jobs only in warp 3, 36 of them: two rounds of warp 0's lanes
             [FAR, mid(), mid(), mid()] +       # none in warp 0
             [DEEP] * 4 +                       # 4 x 36 jobs: five rounds
             [mid(), DEEP, mid(), FAR] +
             [rs.uniform(0.004, 0.12) for _ in range(8)] +
             [mid(), DEEP, mid()])              # 27 envs: the last block has three
    gq = m.jnt_qposadr[-1]
    q = np.tile(m.qpos0, (len(dists), 1))
    for i, dd in enumerate(dists):
        u = rs.normal(size=3)
        q[i, 0:3], q[i, 3:7] = rs.normal(size=3) * 0.01, quat_of(cc.rand_rot(rs))
        q[i, gq:gq + 3], q[i, gq + 3:gq + 7] = q[i, 0:3] + dd * u / np.linalg.norm(u), quat_of(cc.rand_rot(rs))
    return cc.f32(q), dists


def run_batch(m, q, lib_path):
    sim = st.BatchedStepper(m, len(q), lib_path=lib_path)
    sim.reset(q)
    sim.forward()
    return sim.get(st.NCON)[:, 0].astype(int), np.asarray(sim.get(st.CONTACT)).reshape(len(q), -1, 16), sim.get(st.FLAGS)[:, 0]


def gate_env(m, q, ncon, rows, rs, per_pair, name):
    """every pair of one env against orc_pair on the oracle's geom poses, and the contact list against the oracle's forward"""
    o = fo.Oracle(m)
    o.reset(q)
    o.forward()
    ora_all, orow = contacts(o.get(fo.CONTACT), int(o.get(fo.NCON)[0]))
    dev_all, drow = contacts(rows, ncon)
    assert np.array_equal(drow[:, 7:9], orow[:, 7:9]) or len(drow) != len(orow) or name is None, (name, drow[:, 7:9], orow[:, 7:9])
    poses = body_poses(m, q)
    for g1, g2 in zip(m.pair_geom1, m.pair_geom2):
        c = pair_case(m, poses, g1, g2)
        c.name = f'{name}:{c.name}'
        di = [i for i in range(len(drow)) if (drow[i, 7], drow[i, 8]) == (g1, g2)]
        oi = [i for i in range(len(orow)) if (orow[i, 7], orow[i, 8]) == (g1, g2)]
        judge(c, dev_all[di], ora_all[oi], rs, per_pair.setdefault(c.pair, new_stats()), drow[di, 10], orow[oi, 10])
    return len(orow)


def pooled_gates(title, lib_path=None):
    m = pooled_model()
    q, dists = pooled_batch(m)
    n = len(q)
    ncon, rows, flags = run_batch(m, q, lib_path)
    assert (flags == 0).all(), flags
    rs = np.random.RandomState(23)
    per_pair = {}
    counts = [gate_env(m, q[i], ncon[i], rows[i], rs, per_pair, f'env{i}') for i in range(n)]
    # the job distributions the batch was built for (a contact is a job; FAR envs have no candidate at all)
    blocks = [counts[b:b + FB_WPB] for b in range(0, n, FB_WPB)]
    print(f'\n{title}: oracle contacts per block {blocks}')
    assert n % FB_WPB and blocks[0][:3] == [0, 0, 0] and blocks[0][3] == 36 and blocks[1][0] == 0 and min(blocks[1][1:]) > 0
    assert blocks[2] == [36] * 4 and max(sum(b) for b in blocks) > 32
    table(title, per_pair)
    # bitwise the same contact rows: each env moved to other block neighbours and another warp position, and each env alone
    nb = -(-n // FB_WPB)
    perm = np.array([FB_WPB * ((i // FB_WPB + i % FB_WPB) % nb) + (i % FB_WPB + 1) % FB_WPB for i in range(n)])   # env i runs as perm[i]
    perm[perm >= n] = sorted(set(range(n)) - set(perm.tolist()))          # the ragged block: into the slot left free
    assert sorted(perm.tolist()) == list(range(n))
    assert all(perm[i] % FB_WPB != i % FB_WPB for i in range(n)) and all(
        perm[i] // FB_WPB != perm[j] // FB_WPB for i in range(n) for j in range(n) if i != j and i // FB_WPB == j // FB_WPB)
    qp = np.empty_like(q)
    qp[perm] = q
    ncon_p, rows_p, _ = run_batch(m, qp, lib_path)
    for i in range(n):
        assert ncon_p[perm[i]] == ncon[i] and np.array_equal(rows_p[perm[i]].view(np.uint32), rows[i].view(np.uint32)), ('permuted', i)
        nc1, rows1, _ = run_batch(m, q[i:i + 1], lib_path)
        assert nc1[0] == ncon[i] and np.array_equal(rows1[0].view(np.uint32), rows[i].view(np.uint32)), ('alone', i)


def test_pooled_mpr_jobs_under_emulation():
    """the same batches on the kernel source (which runs each env's jobs on its own warp): the gates and the bitwise comparisons"""
    ge.build()
    pooled_gates('pooled MPR batch (emulation)', lib_path=ge.EMU)


@pytest.mark.gpu
def test_pooled_mpr_jobs_on_gpu():
    """kcol_mpr's pooled path: warp 0 runs the MPR jobs of all four envs of its block, reading the other warps' shared slices"""
    pooled_gates('pooled MPR batch (H100)')


# --------------------------------------------------------------------------------------------------------------- d. capacities

FB_MAXCAND, FB_MAXCON = 192, 64


def capsule_grid(k, touching, lift):
    """k capsules on the thorax along x, k on the ghost along y spread over x, the ghost `lift` above the thorax.  The thorax capsules
    i in `touching` lie at height 0 and touch every ghost capsule (axes 0.012 apart, radii 0.008); the others lie 0.03 above or
    below, where every pair still passes the broadphase but none touches"""
    z_to_x, z_to_y = [np.cos(np.pi / 4), 0, np.sin(np.pi / 4), 0], [np.cos(np.pi / 4), -np.sin(np.pi / 4), 0, 0]
    size = [0.008, 0.03, 0]
    m = multi_model([cc.CAP] * k, [size] * k, [cc.CAP] * k, [size] * k,
                    pos1=[[0, 0, 0.0 if i in touching else 0.03 * (1 if i % 2 else -1)] for i in range(k)], quat1=[z_to_x] * k,
                    pos2=[[0.004 * j - 0.002 * (k - 1), 0, 0] for j in range(k)], quat2=[z_to_y] * k)
    q = m.qpos0.copy()
    gq = m.jnt_qposadr[-1]
    q[0:3], q[3:7], q[gq:gq + 3], q[gq + 3:gq + 7] = 0, [1, 0, 0, 0], [0, 0, lift], [1, 0, 0, 0]
    return m, cc.f32(q)


def capacity_gates(title, lib_path=None):
    rs = np.random.RandomState(29)
    for name, (k, touching, lift), want_cand, want_con in (('candidates', (15, (5, 12), 0.012), 225, 30), ('contacts', (9, range(9), 0.012), 81, 81)):
        m, q = capsule_grid(k, touching, lift)
        poses = body_poses(m, q)
        # the oracle's broadphase in numpy (bounding spheres), in pair order; the kernel keeps the first 192 candidates
        cand = [(g1, g2) for g1, g2 in zip(m.pair_geom1, m.pair_geom2)
                if np.sum((poses[g2][0] - poses[g1][0]) ** 2) <= (max(m.geom_margin[g1], m.geom_margin[g2]) + m.geom_rbound[g1] + m.geom_rbound[g2]) ** 2]
        full = [(g1, g2, con) for g1, g2 in cand for con in pair_case(m, poses, g1, g2).oracle()]
        assert (len(cand), len(full)) == (want_cand, want_con), (name, len(cand), len(full))
        kept = [(g1, g2, con) for g1, g2 in cand[:FB_MAXCAND] for con in pair_case(m, poses, g1, g2).oracle()][:FB_MAXCON]
        ncon, rows, flags = run_batch(m, q[None], lib_path)
        dev, drow = contacts(rows[0], ncon[0])
        print(f'\n{title} {name}: {len(cand)} candidates, {len(full)} contacts, {len(kept)} kept; device ncon {ncon[0]}, FLAGS {int(flags[0])}')
        assert int(flags[0]) & 2, flags
        assert ncon[0] == len(kept) and [(int(a), int(b)) for a, b in drow[:, 7:9]] == [(g1, g2) for g1, g2, _ in kept]
        per_pair = {}
        for i, (g1, g2, con) in enumerate(kept):
            c = pair_case(m, poses, g1, g2)
            judge(c, dev[i:i + 1], con[None], rs, per_pair.setdefault(c.pair, new_stats()))
        table(f'{title} {name}', per_pair)


def test_capacities_under_emulation():
    """more than FB_MAXCAND = 192 broadphase candidates, and more than FB_MAXCON = 64 contacts: the overflow flag, and the kept
    contacts are the oracle's of the first 192 candidates, the first 64 of them, in pair order"""
    ge.build()
    capacity_gates('capacities (emulation)', lib_path=ge.EMU)


@pytest.mark.gpu
def test_capacities_on_gpu():
    capacity_gates('capacities (H100)')
