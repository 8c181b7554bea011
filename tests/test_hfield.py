"""Convex geom against a heightfield (MuJoCo mjc_ConvexHField): the fp64 oracle (`orc_convex_hfield`) against closed forms, and the
`vision` model's forward pass on a terrain against the oracle.  The device code (`fb_hfield.h`) is gated prism by prism and contact by
contact in tests/test_hfield_gates.py."""
import ctypes as C

import numpy as np
import pytest

import __graft_entry__ as ge
from oracle import fly_oracle as fo
from test_oracle_invariants import SPH, _rot

dp = lambda a: np.ascontiguousarray(a, np.float64).ctypes.data_as(C.POINTER(C.c_double))
EYE = np.eye(3)


@pytest.fixture(scope='module')
def libs():
    ge.build()
    o = C.CDLL(fo.build())
    o.orc_convex_hfield.argtypes = [C.c_int] + [C.POINTER(C.c_double)] * 3 + [C.c_double] + [C.POINTER(C.c_double)] * 3 + [C.c_int, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_int]
    return o


def oracle_hf(o, t, p, R, s, margin, hp, hR, hsize, data, kmax=50):
    out = np.zeros((kmax, 7))
    n = o.orc_convex_hfield(t, dp(p), dp(np.asarray(R).reshape(9)), dp(s), margin, dp(hp), dp(np.asarray(hR).reshape(9)), dp(hsize), data.shape[0], data.shape[1],
                            dp(data), dp(out), kmax)
    return out[:n]


HSIZE = np.array([2.0, 2.0, 1.0, 0.05])            # 4 x 4 arena, elevation scale 1, base 0.05
GRID = 41                                           # 0.1 spacing, as the flight arenas (hills.py:172-176)


def test_oracle_sphere_on_flat_and_tilted_terrain(libs):
    o = libs
    flat = np.full((GRID, GRID), 0.3)
    r = 0.04
    for z, hit in ((0.3 + r - 0.004, True), (0.3 + r + 0.003, False)):
        c = oracle_hf(o, SPH, [0.13, -0.21, z], EYE, [r, 0, 0], 0.0, [0, 0, 0], EYE, HSIZE, flat)
        assert (len(c) > 0) == hit
        if hit:
            k = np.argmin(c[:, 0])
            assert abs(c[k, 0] - (z - r - 0.3)) < 2e-6 and np.allclose(c[k, 4:], [0, 0, 1], atol=1e-4)       # the plane-sphere answer
            assert np.all(c[:, 0] >= c[k, 0] - 1e-9) and np.all(c[:, 6] > 0.5)
    # margin: reported from margin away, dist stays the geometric distance
    c = oracle_hf(o, SPH, [0.13, -0.21, 0.3 + r + 0.003], EYE, [r, 0, 0], 0.01, [0, 0, 0], EYE, HSIZE, flat)
    assert len(c) > 0 and abs(c[:, 0].min() - 0.003) < 2e-6
    # a plane of slope b along x: distance (z - H(x)) cos(theta) - r, normal (-sin, 0, cos)
    b = 0.25
    xs = np.linspace(-2, 2, GRID)
    ramp = np.tile(0.5 + b * xs / 1.0, (GRID, 1)) / 1.0
    th = np.arctan(b)
    x0, z0 = 0.31, 0.5 + b * 0.31 + 0.035 / np.cos(th)                       # 0.005 cos(theta) deep
    c = oracle_hf(o, SPH, [x0, 0.17, z0], EYE, [r, 0, 0], 0.0, [0, 0, 0], EYE, HSIZE, ramp)
    k = np.argmin(c[:, 0])
    assert abs(c[k, 0] - ((z0 - (0.5 + b * x0)) * np.cos(th) - r)) < 5e-6
    assert np.allclose(c[k, 4:], [-np.sin(th), 0, np.cos(th)], atol=2e-3)
    # the heightfield's own frame: the same scene rotated and shifted as a whole gives the same distances
    R = _rot(np.random.RandomState(1))
    t = np.array([0.4, -0.7, 0.2])
    c2 = oracle_hf(o, SPH, R @ np.array([x0, 0.17, z0]) + t, R, [r, 0, 0], 0.0, t, R, HSIZE, ramp)
    assert len(c2) == len(c) and np.allclose(np.sort(c2[:, 0]), np.sort(c[:, 0]), atol=1e-6)
    k2 = np.argmin(c2[:, 0])
    assert np.allclose(c2[k2, 4:], R @ c[k, 4:], atol=1e-5) and np.allclose(c2[k2, 1:4], R @ c[k, 1:4] + t, atol=1e-5)
    # outside the footprint or above the tallest point: nothing
    assert len(oracle_hf(o, SPH, [2.2, 0, 0.3], EYE, [r, 0, 0], 0.0, [0, 0, 0], EYE, HSIZE, flat)) == 0
    assert len(oracle_hf(o, SPH, [0, 0, 1.2], EYE, [r, 0, 0], 0.0, [0, 0, 0], EYE, HSIZE, flat)) == 0


def test_vision_model_terrain_contacts_match_the_oracle_through_the_step():
    check_vision_terrain_contacts(ge.EMU)


def check_vision_terrain_contacts(lib):
    """the compiled `vision` variant (flight model, no ghost, ground contacts on, 401 x 401 terrain geom): stage parity of the whole
    forward pass against the oracle with the fly dipped into a bumpy terrain -- heightfield contacts, their rows and forces."""
    import __graft_entry__ as ge
    from flybody_b200 import arenas, stepper as st
    from flybody_b200.flymodel import load_model
    from parity_common import rel_err
    ge.build()
    m = load_model('vision')
    assert (m.nq, m.nv, m.nu) == (43, 42, 11) and m.meta['hf_nrow'] == 401 and len(m.hf_pair_geom) == 70
    terr = arenas.SineBumps().generate(np.random.RandomState(4)).astype(np.float32)
    rs = np.random.RandomState(0)
    for trial, dz in enumerate((0.13, 0.17, 0.6)):
        x, y = (-5.0, 0.0) if trial < 2 else (3.0, -2.0)
        ground = float(arenas.hfield_height(terr, [x], [y], 20.0)[0]) - 0.01
        q = m.qpos0.copy(); q[:3] = [x, y, ground + dz]
        v = np.zeros(m.nv); v[0] = 20.0
        sim = st.BatchedStepper(m, 2, lib_path=lib)
        sim.hfield_collision(m.meta['hf_geom'], m.hf_size, 401, 401, m.hf_pair_geom)
        sim.hfield_write(np.arange(2), np.stack([terr, terr]))
        o = fo.Oracle(m, tolerance=1e-12)
        o.set_hfield(m.meta['hf_geom'], m.hf_size, terr, m.hf_pair_geom)
        ctrl = rs.uniform(-0.2, 0.2, m.nu)
        o.reset(q, v); sim.reset(np.tile(q, (2, 1)), np.tile(v, (2, 1)))
        o.set(fo.CTRL, ctrl); sim.set_control(np.tile(ctrl, (2, 1)).astype(np.float32))
        o.forward(); sim.forward()
        ncon_o, ncon_d = int(o.get(fo.NCON)[0]), int(sim.get(st.NCON)[1, 0])
        co = o.get(fo.CONTACT).reshape(-1, 16)[:ncon_o]
        terrain_contacts = int((co[:, 7] == m.meta['hf_geom']).sum())
        assert (terrain_contacts > 0) == (dz < 0.3), (trial, terrain_contacts)
        assert ncon_o == ncon_d and int(o.get(fo.NEFC)[0]) == int(sim.get(st.NEFC)[1, 0])
        cd = sim.get(st.CONTACT)[1].reshape(-1, 16)[:ncon_d].astype(np.float64)
        assert np.array_equal(co[:, 7:9], cd[:, 7:9])                                   # same geom pairs in the same order
        assert np.abs(co[:, 0] - cd[:, 0]).max() < 5e-5                                 # distances
        for f in (fo.EFC_FORCE, fo.QFRC_CONSTRAINT, fo.QACC):
            a = o.get(f)
            if np.abs(a).max() > 0:
                assert rel_err(a, sim.get(f)[1]) < 2e-3, (trial, f)
        sim.close()


def test_vision_model_stage_parity_in_free_flight():
    check_vision_free_flight(ge.EMU)


def check_vision_free_flight(lib):
    """the `vision` variant away from the ground: every stage of the forward pass against the oracle (as the flight variant)."""
    import __graft_entry__ as ge
    from flybody_b200 import stepper as st
    from flybody_b200.flymodel import load_model
    from parity_common import compare_stage_fields
    ge.build()
    m = load_model('vision')
    res = compare_stage_fields(m, st.BatchedStepper(m, 2, lib_path=lib), seed=1, vel_scale=20.0)
    assert 'qM' in res and 'qfrc_passive' in res
