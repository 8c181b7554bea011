"""Pinned heightfield cases for tests/test_hfield_gates.py: one convex geom (sphere, capsule, ellipsoid, cylinder) against a
heightfield, on flat, ramped (along x, y and both diagonals, which cut a cell's two triangles differently), sine-bump, trench, single
raised / pit vertex and step terrains, in identity, shifted, rotated and near-upright terrain frames, with named placements at the
grid's edges.

A case holds the geom's and the terrain's poses, the sizes and the heights rounded to fp32 (what the stepper holds), so that the oracle
and the kernel source see the same numbers.  Depths are placed with the oracle (`orc_convex_hfield`) by bisection along the terrain's
up axis, so a random case sits at a known oracle distance between -0.3 rbound and margin + 1e-3.
"""
import ctypes as C
from dataclasses import dataclass, field

import numpy as np

from collision_cases import f32, rot_axis, rand_rot, EYE
from flybody_b200 import arenas
from flybody_b200.compiler.compile_model import rbound
from oracle import fly_oracle as fo

SPH, CAP, ELL, CYL = 2, 3, 4, 5
NAMES = {SPH: 'sphere', CAP: 'capsule', ELL: 'ellipsoid', CYL: 'cylinder'}
TYPES = (SPH, CAP, ELL, CYL)
MARGINS = ((0.0, 0.0), (0.01, 0.005))          # (margin, gap)
SMALL = (41, [2.0, 2.0, 1.0, 0.05])           # 41 x 41 over +-2: 0.1 cells, as the flight arenas
VISION = (401, [20.0, 20.0, 1.0, 0.05])       # the `vision` model's 401 x 401 over +-20
# the `vision` model's geom sizes (fly_vision.npz: hf_pair_geom) and a few larger ones
SIZES = {SPH: [[0.00788, 0, 0], [0.05, 0, 0]],
         CAP: [[0.0035, 0.0127195, 0], [0.00481, 0.00875, 0], [0.03, 0.06, 0]],
         ELL: [[0.0437, 0.0437, 0.0551], [0.0131, 0.0219, 0.0131], [0.06, 0.1, 0.04]],
         CYL: [[0.0035, 0.00875, 0.0131], [0.02, 0.05, 0]]}
NEAR_UPRIGHT = (1e-4, 1e-3, 5e-3, 1.4e-2)     # yaw / tilt of the near-upright terrain frames (rad)


_LIB = None


def oracle_lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(fo.build())
        _LIB.orc_convex_hfield_prisms.argtypes = [C.c_int] + [C.c_void_p] * 3 + [C.c_double] + [C.c_void_p] * 3 + [C.c_int, C.c_int] + [C.c_void_p] * 2 + [C.c_int, C.c_void_p]
    return _LIB


def oracle_hf(t, p, R, s, margin, hp, hR, hsize, data, kmax=50):
    """fp64 contacts [n, 7] (dist, pos, normal) and their prism ids [n]"""
    d = lambda a: np.ascontiguousarray(a, np.float64)
    args = [d(p), d(np.asarray(R).reshape(9)), d(s), None, d(hp), d(np.asarray(hR).reshape(9)), d(hsize), None, None, d(data)]
    out, pr = np.zeros((kmax, 7)), np.zeros(kmax, np.int32)
    n = oracle_lib().orc_convex_hfield_prisms(t, args[0].ctypes.data, args[1].ctypes.data, args[2].ctypes.data, float(margin), args[4].ctypes.data,
                                              args[5].ctypes.data, args[6].ctypes.data, data.shape[0], data.shape[1], args[9].ctypes.data,
                                              out.ctypes.data, kmax, pr.ctypes.data)
    return out[:n], pr[:n]


# ------------------------------------------------------------------------------------------------------------------- terrains

def _axes(n, half):
    return np.linspace(-half, half, n)


def terrains():
    """{name: (heights [n, n] fp32-rounded, hsize)}"""
    T = {}
    n, hs = SMALL
    x = _axes(n, hs[0])
    X, Y = np.meshgrid(x, x)                    # row = y, column = x
    T['flat0'] = (np.zeros((n, n)), hs)
    T['flat1'] = (np.ones((n, n)), hs)
    for s in (0.05, 0.5, 3.0):
        for name, u in (('x', X), ('y', Y), ('d1', (X + Y) / np.sqrt(2)), ('d2', (X - Y) / np.sqrt(2))):
            T[f'ramp_{name}_{s:g}'] = (0.5 + s * u, hs)
    v = np.full((n, n), 0.3)
    v[20, 21] = 0.45
    T['raised_vertex'] = (v, hs)
    v = np.full((n, n), 0.3)
    v[20, 21] = 0.15
    T['pit_vertex'] = (v, hs)
    v = np.zeros((n, n))
    v[21:] = 1.0
    T['step'] = (v, hs)                         # rows 20 -> 21 (y = 0 -> 0.1): 0 -> 1
    nv, hv = VISION
    T['bumps'] = (arenas.SineBumps().generate(np.random.RandomState(4)).astype(np.float64), hv)
    T['trench'] = (arenas.SineTrench().generate(np.random.RandomState(6)).astype(np.float64), hv)
    return {k: (f32(h), f32(s)) for k, (h, s) in T.items()}


def height(data, hsize, x, y):
    """the terrain's surface under (x, y) of its frame: the strip's triangles (split along (c, r + 1) - (c + 1, r))"""
    n, m = data.shape
    fx, fy = (x + hsize[0]) / (2 * hsize[0]) * (m - 1), (y + hsize[1]) / (2 * hsize[1]) * (n - 1)
    c, r = int(np.clip(np.floor(fx), 0, m - 2)), int(np.clip(np.floor(fy), 0, n - 2))
    u, v = fx - c, fy - r
    h00, h10, h01, h11 = data[r, c], data[r, c + 1], data[r + 1, c], data[r + 1, c + 1]
    z = h00 + u * (h10 - h00) + v * (h01 - h00) if u + v <= 1 else h11 + (1 - u) * (h01 - h11) + (1 - v) * (h10 - h11)
    return z * hsize[2]


# ---------------------------------------------------------------------------------------------------------------------- cases

def frames(rs):
    """(name, hp, hR) terrain frames: identity, shifted, an arbitrary rotation, near-upright yaws and tilts"""
    out = [('identity', np.zeros(3), EYE), ('shifted', np.array([0.31, -0.27, 0.12]), EYE),
           ('rotated', np.array([0.2, -0.1, -0.01]), rand_rot(np.random.RandomState(17)))]
    for a in NEAR_UPRIGHT:
        out.append((f'yaw{a:g}', np.array([0.05, 0.0, -0.01]), rot_axis([0, 0, 1], a)))
        out.append((f'tilt{a:g}', np.array([0.0, 0.05, -0.01]), rot_axis([1, 0.3, 0], a)))
    return out


@dataclass
class HCase:
    name: str
    t: int
    p: np.ndarray
    R: np.ndarray
    s: np.ndarray
    margin: float
    gap: float
    hp: np.ndarray
    hR: np.ndarray
    terrain: str
    data: np.ndarray = field(repr=False)
    hsize: np.ndarray = field(repr=False)
    kmax: int = 50
    check: object = field(default=None, repr=False)

    def __post_init__(self):
        for k in ('p', 'R', 's', 'hp', 'hR', 'hsize'):
            setattr(self, k, f32(getattr(self, k)))
        self.margin, self.gap = float(np.float32(self.margin)), float(np.float32(self.gap))

    @property
    def rb(self):
        return rbound(self.t, self.s)

    @property
    def pos_scale(self):
        """the device adds the geom's offset from the terrain's origin back in fp32: its resolution in position"""
        return max(self.rb, float(np.linalg.norm(self.p - self.hp)))

    def oracle(self, kmax=None, p=None, R=None):
        return oracle_hf(self.t, self.p if p is None else p, self.R if R is None else R, self.s, self.margin, self.hp, self.hR, self.hsize,
                         self.data, self.kmax if kmax is None else kmax)

    def moved(self, name, **kw):
        d = dict(self.__dict__)
        d.update(name=name, **kw)
        return HCase(**d)


def oracle_dist(c, margin):
    con, _ = c.moved(c.name, margin=margin).oracle()
    return float(con[:, 0].min()) if len(con) else np.inf


def place(t, s, R_local, x, y, target, margin, gap, hp, hR, name, tname, data, hsize, below=None):
    """the geom at (x, y) of the terrain frame, rotated by R_local in it, lifted along the terrain's up axis until the oracle's smallest
    dist is `target` (placed with the margin widened: a prism's dist hardly depends on it); the search starts `below` (default 2 rbound)
    under the surface"""
    rb = rbound(t, np.asarray(s, np.float64))
    z0 = height(data, hsize, x, y)
    base = HCase(name, t, hp, hR @ R_local, s, margin, gap, hp, hR, tname, data, hsize)
    at = lambda z: base.moved(name, p=hp + hR @ np.array([x, y, z]))
    lo, hi = z0 - (2 * rb if below is None else below), z0 + float(np.ptp(data)) * hsize[2] + 2 * rb + 0.05
    wide = margin + max(0.0, target - margin) + 2e-3
    for _ in range(60):
        mid = 0.5 * (lo + hi)
        lo, hi = (mid, hi) if oracle_dist(at(mid), wide) < target else (lo, mid)
    return at(0.5 * (lo + hi))


def random_cases(rs, t, tname, data, hsize, n, frame_list, tag='random', xy=None):
    out = []
    for i in range(n):
        s = SIZES[t][i % len(SIZES[t])]
        margin, gap = MARGINS[i % 2]
        fname, hp, hR = frame_list[i % len(frame_list)]
        rb = rbound(t, np.asarray(s, np.float64))
        lim = 0.99 * hsize[0] - rb
        x, y = xy(rs) if xy is not None else rs.uniform(-min(lim, 1.7), min(lim, 1.7), 2)
        target = rs.uniform(-0.3 * rb, margin + 1e-3)
        out.append(place(t, s, rand_rot(rs), x, y, target, margin, gap, hp, hR, f'{tag}{i}_{tname}_{fname}', tname, data, hsize))
    return out


def _expect(cond, msg):
    if not cond:
        raise AssertionError(msg)


def edge_cases(T):
    """named placements, each with the property that makes it an edge (asserted by `check`)"""
    E = []
    data, hs = T['flat0']
    dx = 2 * hs[0] / (data.shape[1] - 1)
    for t in TYPES:
        s = SIZES[t][0]
        rb = rbound(t, np.asarray(s, np.float64))
        R0 = rot_axis([1, 0.5, 0.2], 0.7)
        for where, (x, y) in (('cell_interior', (0.031, 0.047)), ('cell_edge', (0.05, 0.0)), ('diagonal', (0.03, 0.07)),
                              ('vertex', (0.1, -0.2)), ('straddle_x+', (hs[0] - 0.3 * rb, 0.3)), ('straddle_x-', (-hs[0] + 0.3 * rb, -0.4)),
                              ('straddle_y+', (0.2, hs[1] - 0.3 * rb)), ('straddle_y-', (-0.6, -hs[1] + 0.3 * rb)),
                              ('corner', (hs[0] - 0.3 * rb, -hs[1] + 0.3 * rb))):
            for tn in ('flat0', 'ramp_x_0.5', 'ramp_d1_0.5', 'ramp_d2_0.5'):
                d, h = T[tn]
                E.append(place(t, s, R0, x, y, -0.1 * rb, 0.0, 0.0, np.zeros(3), EYE, f'{where}_{tn}_{NAMES[t]}', tn, d, h))
        # the bounding box's low x and y edges exactly on grid lines (x = 0.5, y = -1) (a sphere: lo.x = x - r, in fp32 and fp64 alike)
        if t == SPH:
            r = float(np.float32(0.0625))
            c = place(t, [r, 0, 0], EYE, 0.5 + r, -1.0 + r, -0.01, 0.0, 0.0, np.zeros(3), EYE, 'bbox_on_grid_lines', 'flat0', data, hs)
            c = c.moved(c.name, p=np.array([0.5 + r, -1.0 + r, c.p[2]]), s=np.array([r, 0, 0]))

            def on_grid(c, con):
                fx = (c.p[0] - c.s[0] + c.hsize[0]) / (2 * c.hsize[0]) * (c.data.shape[1] - 1)
                _expect(abs(fx - round(fx)) < 1e-9 and len(con) > 0, f'{c.name}: {fx}')
            E.append(c.moved(c.name, check=on_grid))
        # 1e-4 beyond the border, and above the highest point: no contact
        # (axis z, unrotated: the geom's half extent along x is its radius, an ellipsoid's first semi-axis)
        def beyond_border(c, con):
            _expect(len(con) == 0 and abs(c.p[0] - c.s[0] - c.hsize[0] - 1e-4) < 1e-6, f'{c.name}: {len(con)} contacts')
        E.append(HCase(f'beyond_border_{NAMES[t]}', t, [float(np.float32(hs[0] + s[0] + 1e-4)), 0.1, 0.0], EYE, s, 0.0, 0.0, np.zeros(3), EYE,
                       'flat0', data, hs, check=beyond_border))
        d1, h1 = T['ramp_x_0.5']
        top = float(d1.max()) * h1[2]
        E.append(HCase(f'above_highest_{NAMES[t]}', t, [1.9, 0.0, top + rb + 1e-3], rot_axis([0, 1, 0], 0.3), s, 0.0, 0.0, np.zeros(3), EYE,
                       'ramp_x_0.5', d1, h1, check=lambda c, con: _expect(len(con) == 0, c.name)))
        # dist = margin -/+ 1e-6 on both margin settings
        for margin, gap in MARGINS:
            for side, off in (('below', -1e-6), ('above', 1e-6)):
                want = margin + off
                c = place(t, s, R0, 0.237, -0.113, want, margin, gap, np.zeros(3), EYE, f'margin_{side}_m{margin:g}_{NAMES[t]}', 'ramp_y_0.05',
                          *T['ramp_y_0.05'])

                def at_margin(c, con, want=want):
                    d = oracle_dist(c, c.margin + 2e-3)
                    _expect(abs(d - want) < 2e-7, f'{c.name}: oracle dist {d}, want {want}')      # (either decision: MPR's tolerance is 1e-6)
                E.append(c.moved(c.name, check=at_margin))
    return E


def cap_cases(T):
    """a lying capsule and a lying cylinder across six or more prisms of the flat and a ramped terrain, for the 4-per-geom cap"""
    out = []
    for tn in ('flat0', 'ramp_d2_0.05'):
        d, h = T[tn]
        for t, s in ((CAP, [0.02, 0.3, 0]), (CYL, [0.03, 0.3, 0])):
            for axis in ([1, 0, 0], [1, 1, 0]):
                R = rot_axis([-axis[1], axis[0], 0], np.pi / 2 - 1e-2)       # axis z onto `axis`, 1e-2 rad off flat
                out.append(place(t, s, R, 0.013, -0.021, -0.006, 0.01, 0.005, np.zeros(3), EYE, f'lying_{NAMES[t]}_{tn}_{axis[1]}', tn, d, h, below=0.04))
    return out


def all_cases(seed=0, n_random=6):
    """{geom type: [cases]}: random placements on every terrain and frame, far out on the 401 x 401 grid, and the named edges"""
    rs = np.random.RandomState(seed)
    T = terrains()
    fr = frames(rs)
    out = {t: [] for t in TYPES}
    for tn, (data, hs) in T.items():
        for t in TYPES:
            if hs[0] > 10:      # the 401 x 401 terrains: anywhere, out to 0.99 of the half size
                out[t] += random_cases(rs, t, tn, data, hs, n_random, fr, xy=lambda rs: rs.uniform(-19.8, 19.8, 2))
            else:
                out[t] += random_cases(rs, t, tn, data, hs, n_random, fr)
    for c in edge_cases(T):
        out[c.t].append(c)
    return out
