"""Pinned collision cases for tests/test_collision_gates.py: one generator per pair type of the narrowphase dispatch (plane x
{sphere, capsule, cylinder, ellipsoid}, and the 10 pairs of {sphere, capsule, ellipsoid, cylinder}, the generic ones through MPR), and
named edge cases, each with the property that makes it an edge.

A case holds both geoms' poses and sizes rounded to fp32 (what the stepper holds), so that the oracle and the kernel source see the same
numbers.  A plane is geom 1 at the origin with normal +z.  Depths are placed with the oracle (fly_oracle.pair) by bisection along a
direction, so a random case sits at a known oracle distance between -0.3 r and margin + 1e-3.
"""
from dataclasses import dataclass, field

import numpy as np

from flybody_b200.compiler.compile_model import rbound
from oracle import fly_oracle as fo

PLANE, SPH, CAP, ELL, CYL = 0, 2, 3, 4, 5
NAMES = {PLANE: 'plane', SPH: 'sphere', CAP: 'capsule', ELL: 'ellipsoid', CYL: 'cylinder'}
SOLIDS = (SPH, CAP, ELL, CYL)
ANALYTIC = {(PLANE, SPH), (PLANE, CAP), (PLANE, CYL), (PLANE, ELL), (SPH, SPH), (SPH, CAP), (CAP, CAP)}
PAIR_TYPES = [(PLANE, t) for t in (SPH, CAP, CYL, ELL)] + [(a, b) for i, a in enumerate(SOLIDS) for b in SOLIDS[i:]]
MARGINS = ((0.0, 0.0), (5e-4, 5e-4))      # (margin, gap): the walk model's two settings
EYE = np.eye(3)
NEAR = 2e-5                                # prefilter cases: oracle dist within margin -/+ this


def f32(x):
    return np.asarray(x, np.float64).astype(np.float32).astype(np.float64)


def rot_axis(axis, th):
    """rotation by th about the unit axis (Rodrigues)"""
    a = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return EYE + np.sin(th) * K + (1 - np.cos(th)) * K @ K


def rand_rot(rs):
    q = rs.normal(size=4)
    w, x, y, z = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def rand_size(t, rs):
    if t == SPH:
        return [rs.uniform(0.005, 0.05), 0, 0]
    if t in (CAP, CYL):
        return [rs.uniform(0.005, 0.05), rs.uniform(0.005, 0.05), 0]
    return list(rs.uniform(0.005, 0.05, 3))


@dataclass
class Case:
    name: str
    t1: int
    p1: np.ndarray
    R1: np.ndarray
    s1: np.ndarray
    t2: int
    p2: np.ndarray
    R2: np.ndarray
    s2: np.ndarray
    margin: float
    gap: float
    edge: bool = False                  # a named edge case (its property is asserted by `check`)
    check: object = field(default=None, repr=False)

    def __post_init__(self):
        for k in ('p1', 'R1', 's1', 'p2', 'R2', 's2'):
            setattr(self, k, f32(getattr(self, k)))
        self.margin, self.gap = float(np.float32(self.margin)), float(np.float32(self.gap))

    @property
    def pair(self):
        return (self.t1, self.t2)

    @property
    def scale(self):
        """length scale of the pair: the geoms' bounding radii (a radius plus a half length, or the largest semi-axis)"""
        return sum(rbound(t, s) for t, s in ((self.t1, self.s1), (self.t2, self.s2)) if t != PLANE)

    def args(self):
        return (self.t1, self.p1, self.R1, self.s1, self.t2, self.p2, self.R2, self.s2, self.margin)

    def oracle(self):
        return fo.pair(*self.args())

    def moved(self, name, p2=None, R2=None, **kw):
        """a copy with geom 2 moved (and other fields replaced)"""
        d = dict(self.__dict__)
        d.update(name=name, p2=self.p2 if p2 is None else p2, R2=self.R2 if R2 is None else R2, **kw)
        return Case(**d)


def oracle_dist(c):
    con = c.oracle()
    return float(con[:, 0].min()) if len(con) else np.inf


def place(c, u, target, lo=0.0, hi=0.5):
    """geom 2 of `c` moved to p1 + s u (plane: (x, y) kept, height s), with s such that the oracle's smallest dist is `target`"""
    def at(s):
        if c.t1 == PLANE:
            return c.moved(c.name, p2=np.array([c.p2[0], c.p2[1], s]))
        return c.moved(c.name, p2=c.p1 + u * s)
    for _ in range(60):
        mid = 0.5 * (lo + hi)
        lo, hi = (mid, hi) if oracle_dist(at(mid)) < target else (lo, mid)
    return at(0.5 * (lo + hi))


def random_cases(pair, rs, n, sizes=None, margins=MARGINS, depth=None, tag='random'):
    """n cases of one pair type at random poses, alternating the margin settings; depth(rs, case) -> the oracle dist to place at
    (default uniform in [-0.3 r, margin + 1e-3], r the smaller geom's bounding radius); sizes: fixed (s1, s2) for every case"""
    t1, t2 = pair
    out = []
    for i in range(n):
        margin, gap = margins[i % len(margins)]
        s1 = sizes[0] if sizes is not None else ([0, 0, 0] if t1 == PLANE else rand_size(t1, rs))
        s2 = sizes[1] if sizes is not None else rand_size(t2, rs)
        R1 = EYE if t1 == PLANE else rand_rot(rs)
        p1 = np.zeros(3) if t1 == PLANE else rs.normal(size=3) * 0.02
        p2 = np.r_[rs.normal(size=2) * 0.02, 0.0] if t1 == PLANE else p1
        c = Case(f'{tag}{i}', t1, p1, R1, s1, t2, p2, rand_rot(rs), s2, margin, gap)
        r = min(rbound(t, s) for t, s in ((t1, c.s1), (t2, c.s2)) if t != PLANE)
        target = depth(rs, c) if depth is not None else rs.uniform(-0.3 * r, margin + 1e-3)
        u = rs.normal(size=3)
        u /= np.linalg.norm(u)
        # placed with the margin widened, so that a target above the margin is reached too (the dist of a pair does not depend on it)
        wide = place(c.moved(c.name, margin=margin + 2e-3), u, target, lo=-0.5 if t1 == PLANE else 0.0)
        out.append(wide.moved(c.name, margin=margin))
    return out


def prefilter_cases(pair, rs, n):
    """generic pairs whose oracle dist lies within NEAR of the margin on either side: where the prefilter's safety band matters"""
    return random_cases(pair, rs, n, depth=lambda rs, c: c.margin + rs.uniform(-NEAR, NEAR), tag='near')


# ------------------------------------------------------------------------------------------------------------------ edge cases

def _expect(cond, msg):
    if not cond:
        raise AssertionError(msg)


def _count(n):
    def check(c, con):
        _expect(len(con) == n, f'{c.name}: {len(con)} oracle contacts, want {n}')
    return check


def _boundary_cases(pair, s1, s2, R2=EYE, u=(0.0, 0.0, 1.0)):
    """geom 2 placed at oracle dist = margin -/+ 1e-6 (a contact or none) and at dist = margin - gap -/+ 1e-6 (included or not);
    the dist is placed and checked with the margin widened by 1e-3 (an analytic pair's dist does not depend on the margin)"""
    out = []
    base = Case('', pair[0], np.zeros(3), EYE, s1, pair[1], np.zeros(3), R2, s2, 0.0, 0.0)
    for margin, gap in MARGINS:
        for what, edge in (('margin', margin), ('include', margin - gap)):
            for side, off in (('below', -1e-6), ('above', 1e-6)):
                want = edge + off
                c = place(base.moved('', margin=margin + 1e-3), np.asarray(u), want, lo=-0.5 if pair[0] == PLANE else 0.0)

                def check(c, con, want=want):
                    d = oracle_dist(c.moved(c.name, margin=c.margin + 1e-3))
                    _expect(abs(d - want) < 1e-8 and len(con) == int(want <= c.margin), f'{c.name}: oracle dist {d}, want {want}')
                out.append(c.moved(f'{what}_{side}_m{margin:g}', margin=margin, gap=gap, edge=True, check=check))
    return out


def edge_cases():
    """every named edge case, by pair type"""
    E = {}
    r, h = 0.01, 0.03
    E[(SPH, SPH)] = _boundary_cases((SPH, SPH), [0.02, 0, 0], [0.01, 0, 0]) + [
        Case('coincident_centres', SPH, [0.01, -0.02, 0.005], EYE, [0.02, 0, 0], SPH, [0.01, -0.02, 0.005], EYE, [0.01, 0, 0], 0.0, 0.0,
             edge=True, check=lambda c, con: _expect(len(con) == 1 and np.array_equal(con[0, 4:7], [1, 0, 0]) and
                                                    np.array_equal(c.p1, c.p2), c.name))]
    E[(PLANE, SPH)] = _boundary_cases((PLANE, SPH), [0, 0, 0], [0.02, 0, 0])

    # capsule-capsule: the finding of the near-parallel branch (r 0.01, h 0.03, centres 0.015 apart in x and 0.01 in z, capsule 2
    # tilted by th about y)
    def tilted(name, th, check):
        return Case(name, CAP, [0, 0, 0], EYE, [r, h, 0], CAP, [0.015, 0, 0.01], rot_axis([0, 1, 0], th), [r, h, 0], 0.0, 0.0,
                    edge=True, check=check)

    def angle(c):
        a1, a2 = c.R1[:, 2], c.R2[:, 2]
        return float(np.linalg.norm(np.cross(a1, a2)) / (np.linalg.norm(a1) * np.linalg.norm(a2)))

    def non_parallel(th, rel=1e-3):
        def check(c, con):
            _expect(abs(angle(c) - th) < rel * th and len(con) == 1, f'{c.name}: angle {angle(c)}, {len(con)} contacts')
        return check

    cc = [tilted(f'near_parallel_{th:.0e}', th, non_parallel(th)) for th in (1e-2, 1e-3, 1e-4, 1e-5, 1e-6)]
    # the same pair in a rotated frame: the axes' fp32 components then all carry rounding, which moves the angle by up to ~3e-8
    B = rand_rot(np.random.RandomState(5))
    for th in (1e-6, 1e-7):
        t = tilted('', th, None)
        cc.append(Case(f'near_parallel_rotated_{th:.0e}', CAP, B @ t.p1, B @ t.R1, t.s1, CAP, B @ t.p2, B @ rot_axis([0, 1, 0], th),
                       t.s2, 0.0, 0.0, edge=True, check=non_parallel(th, 0.5)))
    cc.append(tilted('parallel', 0.0, lambda c, con: _expect(angle(c) == 0 and len(con) == 2, c.name)))
    # exactly parallel, overlapping lengthwise: two contacts from the parallel branch
    cc.append(Case('parallel_side_by_side', CAP, [0, 0, 0], EYE, [r, h, 0], CAP, [0.019, 0, 0.01], EYE, [r, h, 0], 0.0, 0.0, edge=True,
                   check=_count(2)))

    def clamps(n_clamped):
        def check(c, con):
            x1, x2 = seg_params(c)
            k = int(abs(x1) >= c.s1[1] * (1 - 1e-9)) + int(abs(x2) >= c.s2[1] * (1 - 1e-9))
            _expect(len(con) == 1 and k == n_clamped, f'{c.name}: {k} clamped ends, {len(con)} contacts')
        return check
    cc += [Case('crossing_axes', CAP, [0, 0, 0], EYE, [r, h, 0], CAP, [0.015, 0.005, 0.002], rot_axis([1, 0, 0], np.pi / 2), [r, h, 0],
                0.0, 0.0, edge=True, check=clamps(0)),
           Case('clamped_one_end', CAP, [0, 0, 0], EYE, [r, h, 0], CAP, [0.015, 0.002, 0.036], rot_axis([1, 0, 0], np.pi / 2), [r, h, 0],
                0.0, 0.0, edge=True, check=clamps(1)),
           Case('clamped_both_ends', CAP, [0, 0, 0], EYE, [r, h, 0], CAP, [0.01, 0.0, 0.065], rot_axis([0, 1, 0], 0.7), [r, h, 0],
                5e-4, 5e-4, edge=True, check=clamps(2))]
    cc += _boundary_cases((CAP, CAP), [r, h, 0], [r, h, 0], R2=rot_axis([1, 0, 0], np.pi / 2), u=(1.0, 0.0, 0.0))
    E[(CAP, CAP)] = cc
    E[(SPH, CAP)] = _boundary_cases((SPH, CAP), [0.02, 0, 0], [r, h, 0], u=(1.0, 0.0, 0.0))

    # plane-cylinder: upright (the fallback direction), tilted for 1 / 2 / 4 contacts, lying flat, and the near-upright window
    rc, hc = 0.02, 0.03

    def cyl(name, R, z, check, x=0.0):
        return Case(name, PLANE, [0, 0, 0], EYE, [0, 0, 0], CYL, [x, 0.0, z], R, [rc, hc, 0], 5e-4, 5e-4, edge=True, check=check)

    def upright(c, con):
        a = c.R2[:, 2]
        v = a * (a @ [0, 0, 1.0]) - [0, 0, 1.0]
        _expect(v @ v < 1e-15 and len(con) == 3, f'{c.name}: len2 {v @ v}, {len(con)} contacts')
    pc = [cyl('upright', EYE, hc - 1e-4, upright),
          cyl('upside_down', rot_axis([1, 0, 0], np.pi), hc - 1e-4, upright),
          cyl('tilted_1', rot_axis([1, 0, 0], 0.5), 0.03, _count(1)),
          cyl('tilted_2', rot_axis([1, 0, 0], np.pi / 2 - 0.05), 0.018, _count(2)),
          cyl('tilted_3', rot_axis([1, 0, 0], 0.05), hc - 3e-4, _count(3)),
          cyl('tilted_4', rot_axis([1, 0, 0], 1.4), -0.005, _count(4)),
          # lying flat, 1e-4 rad from exactly flat: at n.axis = 0 the sign of a rounded zero picks the end that gets the contacts
          cyl('lying_flat', rot_axis([1, 0, 0], np.pi / 2 - 1e-4), rc - 2e-4, _count(2)),
          cyl('lying_flat_deep', rot_axis([1, 0, 0], np.pi / 2 - 1e-4), -0.6 * rc, _count(4))]
    for th in (1e-3, 1e-4, 1e-5, 1e-6, 1e-7):
        pc.append(cyl(f'near_upright_{th:.0e}', rot_axis([1, 0, 0], th), hc - 1e-4, _count(3)))
    E[(PLANE, CYL)] = pc
    E[(PLANE, CAP)] = _boundary_cases((PLANE, CAP), [0, 0, 0], [r, h, 0], R2=rot_axis([1, 1, 0], 0.4)) + [
        Case('flat', PLANE, [0, 0, 0], EYE, [0, 0, 0], CAP, [0, 0, r - 1e-4], rot_axis([0, 1, 0], np.pi / 2), [r, h, 0], 0.0, 0.0,
             edge=True, check=_count(2))]

    # plane-ellipsoid: each principal axis along the normal
    se = [0.01, 0.02, 0.035]
    axis_up = [rot_axis([0, 1, 0], np.pi / 2), rot_axis([1, 0, 0], -np.pi / 2), EYE]      # local x, y, z onto world z

    def axis_along(k):
        def check(c, con):
            _expect(abs(abs(c.R2[2, k]) - 1) < 1e-7 and len(con) == 1 and abs(con[0, 3] - c.p2[2] + c.s2[k] + 0.5 * con[0, 0]) < 1e-9,
                    f'{c.name}: {c.R2[2]} {con}')
        return check
    E[(PLANE, ELL)] = [Case(f'axis{k}_along_normal', PLANE, [0, 0, 0], EYE, [0, 0, 0], ELL, [0.003, -0.002, se[k] - 2e-4], axis_up[k],
                            se, 0.0, 0.0, edge=True, check=axis_along(k)) for k in range(3)]

    # generic pairs: shallow, deep, a cylinder rim, and separated by just more than the margin along a principal axis
    for pair in PAIR_TYPES:
        if pair in ANALYTIC:
            continue
        rs = np.random.RandomState(1000 + 10 * pair[0] + pair[1])
        g = []
        for depth, tag in ((-2e-4, 'shallow'), (-0.25, 'deep')):
            c = random_cases(pair, rs, 1, margins=((5e-4, 5e-4),), tag=tag,
                             depth=lambda rs, c, depth=depth: depth if depth > -0.1 else depth * min(rbound(c.t1, c.s1), rbound(c.t2, c.s2)))[0]
            g.append(c.moved(tag, edge=True, check=_count(1)))
        for margin, _ in MARGINS:
            for extra in (2e-5, 5e-6):          # beyond the prefilter's 1e-5 band: pruned; inside it: MPR decides
                g.append(_separated(pair, margin, extra))
        if CYL in pair:
            g.append(_rim(pair))
        E[pair] = g
    return E


def _separated(pair, margin, extra):
    """the geoms' extents along world x (a principal axis of both) separated by margin + extra"""
    t1, t2 = pair
    s1, s2 = [0.012, 0.02, 0.015] if t1 == ELL else [0.012, 0.02, 0], [0.01, 0.03, 0.02] if t2 == ELL else [0.01, 0.03, 0]
    R2 = rot_axis([0, 1, 0], np.pi / 2) if t2 in (CAP, CYL) else EYE       # geom 2's axis along x
    w1 = f32(s1)[0]
    w2 = f32(s2)[0] + (f32(s2)[1] if t2 in (CAP, CYL) else 0) if t2 != ELL else f32(s2)[0]
    x = float(np.float32(w1 + w2 + margin + extra))

    def check(c, con):
        gap = c.p2[0] - w1 - w2
        _expect(len(con) == 0 and abs(gap - margin - extra) < 1e-8, f'{c.name}: gap {gap}, {len(con)} contacts')
    return Case(f'separated_m{margin:g}_{extra:g}', t1, [0, 0, 0], EYE, s1, t2, [x, 0, 0], R2, s2, margin, margin, edge=True, check=check)


def _rim(pair):
    """the contact on a cylinder's rim: geom 1, its longest axis along the approach (a cylinder: across it), pressed 1e-4 deep onto the
    top rim of the cylinder geom 2 (axis z) along the diagonal"""
    t1, t2 = pair
    s1 = [0.01, 0.012, 0.015] if t1 == ELL else [0.01, 0.015, 0]
    R1 = rot_axis([1, 0, 0], np.pi / 2) if t1 == CYL else rot_axis([0, 1, 0], np.pi / 4)
    u = np.array([1.0, 0.0, 1.0]) / np.sqrt(2)
    c = place(Case('rim', t1, [0, 0, 0], R1, s1, t2, [0, 0, 0], EYE, [0.02, 0.025, 0], 5e-4, 5e-4), -u, -1e-4)

    def check(c, con):
        _expect(len(con) == 1, c.name)
        loc = c.R2.T @ (con[0, 1:4] - c.p2)
        _expect(abs(np.hypot(loc[0], loc[1]) - c.s2[0]) < 5e-4 and abs(abs(loc[2]) - c.s2[1]) < 5e-4, f'{c.name}: local {loc}')
    return c.moved('rim', edge=True, check=check)


def seg_params(c):
    """fp64 closest-point parameters (x1, x2) of two capsule axes (MuJoCo's clamping order)"""
    a1, a2, dif = c.R1[:, 2], c.R2[:, 2], c.p1 - c.p2
    ma, mb, mc, u, v = a1 @ a1, -a1 @ a2, a2 @ a2, -a1 @ dif, a2 @ dif
    det = ma * mc - mb * mb
    x1, x2 = (mc * u - mb * v) / det, (ma * v - mb * u) / det
    h1, h2 = c.s1[1], c.s2[1]
    if x1 > h1:
        x1, x2 = h1, (v - mb * h1) / mc
    elif x1 < -h1:
        x1, x2 = -h1, (v + mb * h1) / mc
    if x2 > h2:
        x2, x1 = h2, np.clip((u - mb * h2) / ma, -h1, h1)
    elif x2 < -h2:
        x2, x1 = -h2, np.clip((u + mb * h2) / ma, -h1, h1)
    return x1, x2


def all_cases(n_random=40, n_near=20, seed=0):
    """{pair type: [cases]}: random poses, the prefilter set (generic pairs) and the named edge cases"""
    rs = np.random.RandomState(seed)
    edges = edge_cases()
    out = {}
    for pair in PAIR_TYPES:
        cs = random_cases(pair, rs, n_random)
        if pair not in ANALYTIC:
            cs += prefilter_cases(pair, rs, n_near)
        out[pair] = cs + edges.get(pair, [])
    return out
